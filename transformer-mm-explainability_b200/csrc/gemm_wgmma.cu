// Hopper (sm_90a) tensor-core GEMMs with fp32-faithful numerics:  C[M,N] = A[M,K] * Bt[N,K]^T  (+ epilogue).
//
// The relevancy maps must match the fp32 reference to 1e-4 after ~100 chained GEMMs (forward + dgrad), which rules out
// plain TF32 / fp16 operands.  Each fp32 operand is split exactly into a high and a low part and the product is taken in
// three tensor-core passes, hi*hi + (lo*hi + hi*lo); the dropped lo*lo term is ~2^-21 relative.  Two splits:
//   backend 1, 3xTF32:  hi = x with the low 13 mantissa bits cleared (a TF32 value), lo = x - hi (exact in fp32);
//               wgmma kind tf32 (k = 8 per instruction) on raw fp32 operands, both split inside the kernel.
//   backends 2 / 3, fp16x3:  x = hi + lo' / 2048,  hi = fp16_rn(x),  lo' = fp16_rn((x - hi) * 2048)  (22 significand bits;
//               the 2^11 factor keeps lo' in fp16's normal range); wgmma kind f16 (twice the tf32 rate, k = 16).  The static
//               weights are split ONCE (pack_f16x3) and arrive by TMA ready for the MMAs; backend 2 splits A inside the
//               kernel, backend 3 (the default) in a separate pass before it (split_a_planes_kernel): on H100 the pass costs
//               less than it saves - the kernel then runs a 3-deep ring of pure TMA -> wgmma slabs instead of a 2-deep one
//               with the split in the loop.
// The two cross products go to their OWN accumulator and are folded into the hi*hi accumulator once, in the epilogue,
// with RN: whatever rounding the tensor core applies while accumulating, the cross terms are 2^-11 smaller, and so is
// their share of that error.
//
// Range of fp16x3.  fp16 spans 2^-24 .. 65504: a value above 65504 becomes inf (and the result NaN - loud, never silently
// wrong); values below 2^-14 keep an ABSOLUTE precision of 2^-35, so tensors whose typical magnitude is above ~1e-5 lose
// nothing.  Forward activations and weights of the models on this path sit in 1e-3 .. 1e2.  Gradients do not, which is
// why the CLIP engine normalises the seed gradient of every sample to a power of two near 1 and undoes the factor when
// dA is staged (clip_engine.cu / attention.cu) - an exact operation, and a per-sample one, so batch invariance holds.
//
// Structure: persistent CTAs (at most one per SM) over 128 x BN output tiles, three warpgroups.
//   warps 0-7   two consumer warpgroups, 64 tile rows each: split the slab in shared memory (generic stores, then
//               fence.proxy.async so the tensor core sees them), 3 wgmma per k-group with main and cross accumulators in
//               registers, then the epilogue straight from registers (bias / act' / residual / act; each warp-wide store
//               covers 8 rows x 32 contiguous bytes, whole sectors)
//   warps 8-11  producer warpgroup: one lane fills a ring of STAGES K-slabs by TMA (full / empty mbarriers); the group
//               gives its registers to the consumers (setmaxnreg), whose two accumulators take up to 160 per thread
// A slab is handed back (one arrival per consumer warp on its empty barrier) once wgmma.wait_group shows its MMAs
// retired, so the split of slab k+1 overlaps the MMAs of slab k, and the producer runs ahead into the next tile while the
// consumers store this one.  The tile width BN in {128, 144, 160} is chosen per launch so that the tile count fills
// whole waves of the SMs; every output element sums its K products in the same order whatever BN is, so the choice never
// changes a result bit.
#include "gemm.cuh"
#include "sm90_ptx.cuh"
#include <cuda_fp16.h>
#include <cudaTypedefs.h>
#include <cstdlib>
#include <mutex>

namespace mmx {
namespace wg {

using namespace ::mmx::sm90;

enum Mode { TF32X3 = 0, F16X3 = 1, F16X3_PRESPLIT = 2 };

constexpr int BM = 128;
constexpr int CONSUMER_THREADS = 256, THREADS = CONSUMER_THREADS + 128;
constexpr int REGS_PRODUCER = 40, REGS_CONSUMER = 232;      // 128 x 40 + 256 x 232 <= 64 K registers
constexpr int PLANE_A = BM * 128;              // one 128-row operand plane of 128-byte rows: 16 KB
constexpr float LO_SCALE = 2048.f, LO_INV = 1.f / 2048.f;

template <int MODE, int BN> struct Cfg {
  static_assert(BN % 16 == 0 && BN >= 128 && BN <= 160, "tile width: 128 / 144 / 160");
  static constexpr int BK = MODE == TF32X3 ? 32 : 64;           // one 128-byte row of K per slab and operand plane
  static constexpr int KSTEP = MODE == TF32X3 ? 8 : 16;         // K per wgmma: 32 bytes
  static constexpr int PLANE_B = BN * 128;
  // One ring stage: A hi, A lo, B hi, B lo planes (TF32X3: the raw fp32 tiles land in the hi planes and are split in
  // place), and for the in-kernel fp16 split the raw fp32 A slab as two 32-column boxes behind them.
  static constexpr int OFF_ALO = PLANE_A, OFF_BHI = 2 * PLANE_A, OFF_BLO = 2 * PLANE_A + PLANE_B;
  static constexpr int OFF_ARAW = 2 * PLANE_A + 2 * PLANE_B;
  static constexpr int STAGE = OFF_ARAW + (MODE == F16X3 ? 2 * PLANE_A : 0);
  static constexpr int TX_BYTES = MODE == TF32X3 ? PLANE_A + PLANE_B : 2 * PLANE_A + 2 * PLANE_B;
  static constexpr int FIT = (227 * 1024 - 1024 /*align*/ - 256 /*barriers*/) / STAGE;
  static constexpr int STAGES = FIT > 4 ? 4 : FIT;
  static constexpr int SMEM_BYTES = STAGES * STAGE + 1024 + 256;
  static constexpr int ACC = BN / 2;                              // fp32 registers per thread and accumulator
  static_assert(STAGES >= 2 && SMEM_BYTES <= 227 * 1024, "shared memory per CTA");
};

struct Params {
  int M, N, K, ldc;
  float* C;
  GemmEpilogue ep;
  // batched form (the relevancy updates: one launch for all samples): tile t belongs to sample t / (tiles_m * tiles_n); the
  // operand maps cover the samples stacked along their row dimension (rows_a / rows_b rows per sample), C and the residual
  // advance by stride_c / stride_res elements per sample.  batch = 1: the plain GEMM.
  int batch = 1, rows_a = 0, rows_b = 0;
  long long stride_c = 0, stride_res = 0;
};

// One copy of the activation bodies per kernel (called, not inlined at every store: the erf / exp / tanh bodies are large).
static __device__ __noinline__ float2 act_fwd2(float2 v, int act) { return make_float2(act_fwd(v.x, act), act_fwd(v.y, act)); }
static __device__ __noinline__ float2 act_bwd2(float2 v, int act) { return make_float2(act_bwd(v.x, act), act_bwd(v.y, act)); }

__device__ __forceinline__ void split_tf32(uint32_t& x, uint32_t& lo) {
  const uint32_t h = x & 0xFFFFE000u;
  lo = __float_as_uint(__uint_as_float(x) - __uint_as_float(h));
  x = h;
}
// 16-byte pieces [0, n16) of a raw fp32 plane: hi in place, lo at the same offset of the lo plane (elementwise, so the
// swizzle does not matter)
__device__ __forceinline__ void split_tf32_plane(uint8_t* hi, uint8_t* lo, int n16, int tid, int nthreads) {
  for (int i = tid; i < n16; i += nthreads) {
    uint4 x = reinterpret_cast<const uint4*>(hi)[i], l;
    split_tf32(x.x, l.x); split_tf32(x.y, l.y); split_tf32(x.z, l.z); split_tf32(x.w, l.w);
    reinterpret_cast<uint4*>(hi)[i] = x;
    reinterpret_cast<uint4*>(lo)[i] = l;
  }
}

// (x0, x1) -> packed fp16 pair hi (x0 in the low half: element k of a K-major operand sits below element k+1) and the
// packed pair of the scaled residuals
__device__ __forceinline__ void split2(float x0, float x1, uint32_t& hi, uint32_t& lo) {
  const __half2 h = __floats2half2_rn(x0, x1);
  const float2 hf = __half22float2(h);
  const __half2 l = __floats2half2_rn((x0 - hf.x) * LO_SCALE, (x1 - hf.y) * LO_SCALE);
  hi = *reinterpret_cast<const uint32_t*>(&h);
  lo = *reinterpret_cast<const uint32_t*>(&l);
}
// Rows [r0, r0 + 64) of the raw fp32 A slab (two 128 x 32 boxes, 128-byte swizzle) -> fp16 hi / lo' planes (128 x 64,
// 128-byte swizzle).  Output piece j of row r holds k = 8j .. 8j+7: box j / 4, fp32 pieces 2 (j % 4) and 2 (j % 4) + 1.
__device__ __forceinline__ void split_f16_rows(const uint8_t* raw, uint8_t* hi, uint8_t* lo, int r0, int wtid) {
#pragma unroll
  for (int i = wtid; i < 64 * 8; i += 128) {
    const int r = r0 + (i >> 3), j = i & 7, sw = r & 7, c = 2 * (j & 3);
    const uint8_t* src = raw + (j >> 2) * PLANE_A + r * 128;
    const float4 x0 = *reinterpret_cast<const float4*>(src + ((c ^ sw) << 4));
    const float4 x1 = *reinterpret_cast<const float4*>(src + (((c + 1) ^ sw) << 4));
    uint4 h, l;
    split2(x0.x, x0.y, h.x, l.x);
    split2(x0.z, x0.w, h.y, l.y);
    split2(x1.x, x1.y, h.z, l.z);
    split2(x1.z, x1.w, h.w, l.w);
    const int dst = r * 128 + ((j ^ sw) << 4);
    *reinterpret_cast<uint4*>(hi + dst) = h;
    *reinterpret_cast<uint4*>(lo + dst) = l;
  }
}

template <int MODE, int R>
__device__ __forceinline__ void mma(float (&d)[R], uint64_t a, uint64_t b, uint32_t accumulate) {
  if constexpr (MODE == TF32X3) wgmma_tf32(d, a, b, accumulate);
  else wgmma_f16(d, a, b, accumulate);
}

// map0: A (fp32, or the fp16 hi plane for F16X3_PRESPLIT); map1: the fp16 lo plane of A (F16X3_PRESPLIT only);
// map2: B (fp32 for TF32X3, else the fp16 hi plane); map3: the fp16 lo plane of B (fp16 modes).
template <int MODE, int BN, bool ACT>
__global__ void __launch_bounds__(THREADS, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap map0, const __grid_constant__ CUtensorMap map1,
                  const __grid_constant__ CUtensorMap map2, const __grid_constant__ CUtensorMap map3, Params p) {
  using cfg = Cfg<MODE, BN>;
  constexpr int STAGES = cfg::STAGES, STAGE = cfg::STAGE, BK = cfg::BK, ACC = cfg::ACC;  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;      // swizzle-128B tiles need 1024 B alignment
  uint8_t* smem_gen = smem_raw + (smem_base - smem_u32(smem_raw));
  const uint32_t bar_base = smem_base + STAGES * STAGE;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (STAGES + s); };
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), CONSUMER_THREADS / 32); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (tid == CONSUMER_THREADS) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map0) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map1) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map2) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map3) : "memory");
  }
  __syncthreads();
  // Programmatic dependent launch: everything above touched no global data and may run while the kernel before this one
  // in the stream is still draining; its results (A, the residual, the device-side row count) are read only below.
  pdl_wait();
  if (p.ep.m_dev) p.M = min(p.M, __ldg(p.ep.m_dev));       // ragged batch: the host-side M is only an upper bound
  const int tiles_m = (p.M + BM - 1) / BM, tiles_n = (p.N + BN - 1) / BN;
  const int tiles_per = tiles_m * tiles_n;
  const int num_tiles = tiles_per * p.batch;
  const int nk = (p.K + BK - 1) / BK;

  if (warp >= CONSUMER_THREADS / 32) {
    // ------------------------------------------------------------------ TMA producer (one lane)
    reg_dealloc<REGS_PRODUCER>();
    if (warp == CONSUMER_THREADS / 32 && lane == 0) {
      int stage = 0; uint32_t phase = 0;
      for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
        const int bi = t / tiles_per, tr = t - bi * tiles_per;
        const int ra = bi * p.rows_a + (tr % tiles_m) * BM, rb = bi * p.rows_b + (tr / tiles_m) * BN;   // rows of the stacked maps
        for (int kb = 0; kb < nk; ++kb) {
          mbar_wait(empty_bar(stage), phase ^ 1);
          const uint32_t s = smem_base + stage * STAGE, fb = full_bar(stage);
          const int k0 = kb * BK;
          mbar_expect_tx(fb, cfg::TX_BYTES);
          if constexpr (MODE == TF32X3) {
            tma_load_2d(s, &map0, fb, k0, ra);
            tma_load_2d(s + cfg::OFF_BHI, &map2, fb, k0, rb);
          } else {
            if constexpr (MODE == F16X3) {
              tma_load_2d(s + cfg::OFF_ARAW, &map0, fb, k0, ra);
              tma_load_2d(s + cfg::OFF_ARAW + PLANE_A, &map0, fb, k0 + 32, ra);
            } else {
              tma_load_2d(s, &map0, fb, k0, ra);
              tma_load_2d(s + cfg::OFF_ALO, &map1, fb, k0, ra);
            }
            tma_load_2d(s + cfg::OFF_BHI, &map2, fb, k0, rb);
            tma_load_2d(s + cfg::OFF_BLO, &map3, fb, k0, rb);
          }
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // -------------------------------------------------------------------- consumers: warpgroup wg owns rows 64 wg .. 64 wg + 63
  reg_alloc<REGS_CONSUMER>();
  const int wg = warp >> 2, wtid = tid & 127;
  const uint32_t a_off = (uint32_t)wg * (PLANE_A / 2);
  float acc[ACC], crs[ACC];
#pragma unroll
  for (int i = 0; i < ACC; ++i) { acc[i] = 0.f; crs[i] = 0.f; }
  int stage = 0; uint32_t phase = 0;
  for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
    const int bi = t / tiles_per, tr = t - bi * tiles_per;
    const int m0 = (tr % tiles_m) * BM, n0 = (tr / tiles_m) * BN;
    int prev = -1;
    for (int kb = 0; kb < nk; ++kb) {
      mbar_wait(full_bar(stage), phase);
      uint8_t* sg = smem_gen + stage * STAGE;
      if constexpr (MODE == TF32X3) {
        split_tf32_plane(sg + a_off, sg + cfg::OFF_ALO + a_off, PLANE_A / 2 / 16, wtid, 128);     // own A rows
        split_tf32_plane(sg + cfg::OFF_BHI, sg + cfg::OFF_BLO, cfg::PLANE_B / 16, tid, CONSUMER_THREADS);   // shared B
        fence_proxy_async();
        named_bar_sync(1, CONSUMER_THREADS);
      } else if constexpr (MODE == F16X3) {
        split_f16_rows(sg + cfg::OFF_ARAW, sg, sg + cfg::OFF_ALO, wg * 64, wtid);
        fence_proxy_async();
        named_bar_sync(2 + wg, 128);
      }
      const uint32_t s = smem_base + stage * STAGE;
      const uint64_t a_hi = make_desc(s + a_off), a_lo = make_desc(s + cfg::OFF_ALO + a_off);
      const uint64_t b_hi = make_desc(s + cfg::OFF_BHI), b_lo = make_desc(s + cfg::OFF_BLO);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK / cfg::KSTEP; ++k) {
        const uint64_t adv = (uint64_t)(2 * k);                  // +32 bytes
        const uint32_t first = (kb > 0 || k > 0) ? 1u : 0u;
        mma<MODE>(crs, a_lo + adv, b_hi + adv, first);
        mma<MODE>(crs, a_hi + adv, b_lo + adv, 1u);
        mma<MODE>(acc, a_hi + adv, b_hi + adv, first);
      }
      wgmma_commit();
      wgmma_wait<1>();                                           // the MMAs of the previous slab have retired
      if (prev >= 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(empty_bar(prev));
      }
      prev = stage;
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    fence_regs(acc);
    fence_regs(crs);
    if (prev >= 0) {
      __syncwarp();
      if (lane == 0) mbar_arrive(empty_bar(prev));
    }

    // ------------------------------------------------------------------ epilogue from the accumulator fragments:
    // register 4j + 2h + e holds row 16 (warp % 4) + lane / 4 + 8h, column 8j + 2 (lane % 4) + e of the warpgroup's block.
    // C, pre and residual may alias, so a load written after a store cannot be issued before it: every load of the
    // fragment is written first, into the cross accumulator once it is folded, and the stores come last.  The tile then
    // waits for one memory round trip (two with pre and residual: pre goes first), not one per stored row pair.
    // Arithmetic order per element: fold, + bias, * act'(pre), + residual, store, act(C).
    const int mrow = m0 + wg * 64 + (warp & 3) * 16 + (lane >> 2), cq = 2 * (lane & 3);
    const long long c_off = bi * p.stride_c, r_off = bi * p.stride_res;
    // N % 4 == 0: a column pair is inside or outside
    auto inside = [&](int j, int h) { return n0 + 8 * j + cq < p.N && mrow + 8 * h < p.M; };
    auto load_frag = [&](const float* base, int ld) {            // crs <- base's elements of the thread's fragment
#pragma unroll
      for (int j = 0; j < BN / 8; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h)
          if (inside(j, h)) {
            const float2 x = *reinterpret_cast<const float2*>(base + (long long)(mrow + 8 * h) * ld + n0 + 8 * j + cq);
            crs[4 * j + 2 * h] = x.x; crs[4 * j + 2 * h + 1] = x.y;
          }
    };
#pragma unroll
    for (int i = 0; i < ACC; ++i) {
      if constexpr (MODE == TF32X3) acc[i] = acc[i] + crs[i];
      else acc[i] = fmaf(crs[i], LO_INV, acc[i]);
    }
    if (p.ep.bias) {
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int n = n0 + 8 * j + cq;
        if (n >= p.N) continue;
        const float2 b = __ldg(reinterpret_cast<const float2*>(p.ep.bias + n));
        acc[4 * j] += b.x; acc[4 * j + 1] += b.y; acc[4 * j + 2] += b.x; acc[4 * j + 3] += b.y;
      }
    }
    if (ACT && p.ep.pre) {
      load_frag(p.ep.pre, p.ep.ldpre);
#pragma unroll
      for (int j = 0; j < BN / 8; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h)
          if (inside(j, h)) {
            const int i = 4 * j + 2 * h;
            const float2 f = act_bwd2(make_float2(crs[i], crs[i + 1]), p.ep.act);
            acc[i] *= f.x; acc[i + 1] *= f.y;
          }
    }
    if (p.ep.residual) load_frag(p.ep.residual + r_off, p.ep.ldres);
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const int n = n0 + 8 * j + cq;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (!inside(j, h)) continue;
        const int m = mrow + 8 * h, i = 4 * j + 2 * h;
        float2 v = make_float2(acc[i], acc[i + 1]);
        if (p.ep.residual) { v.x += crs[i]; v.y += crs[i + 1]; }
        if (!ACT || p.ep.C_act != p.C) *reinterpret_cast<float2*>(p.C + c_off + (long long)m * p.ldc + n) = v;
        if (ACT && p.ep.C_act) *reinterpret_cast<float2*>(p.ep.C_act + (long long)m * p.ldc + n) = act_fwd2(v, p.ep.act);
      }
    }
  }
}

// act(fp32 A) [M, K] (row stride lda, lda % 4 == 0) -> hi / lo' fp16 planes [M, ldp]; 4 elements per thread.  Columns
// K .. ldp-1 are never read (the tensor maps declare K columns, TMA zero-fills beyond).  act goes through the epilogue's
// act_fwd2, so act(A) here has the bits a C_act store of the GEMM that produced A would have had.
__global__ void __launch_bounds__(256) split_a_planes_kernel(const float* __restrict__ A, int lda, __half* __restrict__ hi,
                                                             __half* __restrict__ lo, int ldp, int M, int K, int act) {
  const int kc = (K + 3) / 4;
  const long long total = (long long)M * kc;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int m = (int)(i / kc), k = (int)(i % kc) * 4;
    const float* src = A + (long long)m * lda + k;
    float4 x;
    if (k + 4 <= K) x = *reinterpret_cast<const float4*>(src);
    else { x.x = src[0]; x.y = k + 1 < K ? src[1] : 0.f; x.z = k + 2 < K ? src[2] : 0.f; x.w = 0.f; }
    if (act != MMX_ACT_NONE) {
      const float2 a = act_fwd2(make_float2(x.x, x.y), act), b = act_fwd2(make_float2(x.z, x.w), act);
      x = make_float4(a.x, a.y, b.x, b.y);
    }
    uint2 h, l;
    split2(x.x, x.y, h.x, l.x);
    split2(x.z, x.w, h.y, l.y);
    *reinterpret_cast<uint2*>(hi + (long long)m * ldp + k) = h;       // ldp % 8 == 0 and k % 4 == 0: 8-byte aligned, inside the row
    *reinterpret_cast<uint2*>(lo + (long long)m * ldp + k) = l;
  }
}

// fp32 [N,K] (row stride ldw) -> hi / lo' fp16 planes [N, ldp], pad columns K .. ldp-1 zero
__global__ void __launch_bounds__(256) pack_f16x3_kernel(const float* __restrict__ W, int ldw, __half* __restrict__ hi,
                                                         __half* __restrict__ lo, int ldp, int N, int K) {
  const long long total = (long long)N * ldp;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int n = (int)(i / ldp), k = (int)(i % ldp);
    float x = 0.f;
    if (k < K) x = W[(long long)n * ldw + k];
    const __half h = __float2half_rn(x);
    hi[i] = h;
    lo[i] = __float2half_rn((x - __half2float(h)) * LO_SCALE);
  }
}

static PFN_cuTensorMapEncodeTiled_v12000 g_encode = nullptr;   // set by gemm_tc_available()

static int make_map(CUtensorMap* map, CUtensorMapDataType dt, int esize, const void* base, int rows, int K, int ld, int box_k,
                    int box_rows) {
  cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * esize};
  cuuint32_t box[2] = {(cuuint32_t)box_k, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = g_encode(map, dt, 2, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed with code " + std::to_string((int)r));
    return 1;
  }
  return 0;
}

// Tile width for this launch: the BN whose tile count costs the fewest SM-waves x BN (ties and near-ties go to the
// narrower tile).  A ragged launch carries the host's upper bound of the row count; the choice never changes a result bit.
static int pick_bn(int M, int N) {
  const int forced = gemm_tc_tile_n(-1);
  if (forced) return forced;
  const int sms = sm_count(), tiles_m = cdiv(M, BM);
  int best = 128;
  double best_cost = 1e30;
  for (int bn : {128, 144, 160}) {
    const double cost = (double)cdiv(tiles_m * cdiv(N, bn), sms) * bn * (bn == 128 ? 1.0 : 1.04);
    if (cost < best_cost) { best_cost = cost; best = bn; }
  }
  return best;
}

// The operands of one launch: A (fp32, or its fp16 hi plane) with its lo plane for F16X3_PRESPLIT, B (fp32 for TF32X3,
// else the fp16 hi plane) with its lo plane; rows_* = the rows the tensor maps declare (all samples of a batched launch).
struct Operands {
  const void* a; const void* a_lo; int lda, rows_a;
  const void* b; const void* b_lo; int ldb, rows_b;
};

template <int MODE, int BN, bool ACT>
static int launch_kernel(const CUtensorMap (&maps)[4], const Params& p, cudaStream_t st) {
  using cfg = Cfg<MODE, BN>;
  auto kern = gemm_wgmma_kernel<MODE, BN, ACT>;
  // per device: the attribute belongs to the (function, device) pair
  static std::atomic<bool> attr_set[MMX_MAX_DEVICES];
  const int dev = current_device();
  if (!attr_set[dev].load(std::memory_order_acquire)) {
    MMX_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, cfg::SMEM_BYTES));
    attr_set[dev].store(true, std::memory_order_release);
  }
  const int tiles = cdiv(p.M, BM) * cdiv(p.N, BN) * p.batch;
  const int grid = tiles < sm_count() ? tiles : sm_count();
  MMX_CHECK_CUDA(launch_pdl(kern, dim3(grid), dim3(THREADS), cfg::SMEM_BYTES, st, maps[0], maps[1], maps[2], maps[3], p));
  MMX_LAUNCH_CHECK();
  return 0;
}

template <int MODE, int BN>
static int launch_bn(const Operands& o, const Params& p, cudaStream_t st) {
  constexpr int BK = Cfg<MODE, BN>::BK;
  const CUtensorMapDataType fp32 = CU_TENSOR_MAP_DATA_TYPE_FLOAT32, fp16 = CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  CUtensorMap maps[4];
  if (MODE == F16X3_PRESPLIT) {
    MMX_TRY(make_map(&maps[0], fp16, 2, o.a, o.rows_a, p.K, o.lda, BK, BM));
    MMX_TRY(make_map(&maps[1], fp16, 2, o.a_lo, o.rows_a, p.K, o.lda, BK, BM));
  } else {
    MMX_TRY(make_map(&maps[0], fp32, 4, o.a, o.rows_a, p.K, o.lda, 32, BM));
    maps[1] = maps[0];
  }
  if (MODE == TF32X3) {
    MMX_TRY(make_map(&maps[2], fp32, 4, o.b, o.rows_b, p.K, o.ldb, 32, BN));
    maps[3] = maps[2];
  } else {
    MMX_TRY(make_map(&maps[2], fp16, 2, o.b, o.rows_b, p.K, o.ldb, BK, BN));
    MMX_TRY(make_map(&maps[3], fp16, 2, o.b_lo, o.rows_b, p.K, o.ldb, BK, BN));
  }
  if (p.ep.pre || p.ep.C_act) return launch_kernel<MODE, BN, true>(maps, p, st);
  return launch_kernel<MODE, BN, false>(maps, p, st);
}

template <int MODE>
static int launch(const Operands& o, const Params& p, cudaStream_t st) {
  switch (pick_bn(p.M * p.batch, p.N)) {
    case 144: return launch_bn<MODE, 144>(o, p, st);
    case 160: return launch_bn<MODE, 160>(o, p, st);
    default: return launch_bn<MODE, 128>(o, p, st);
  }
}

// the TMA -> wgmma kernel on A already split into fp16 hi / lo' planes [M, ldpa]
static int gemm_planes(const __half* Ahi, const __half* Alo, int ldpa, const BOperand& B, const Params& p, cudaStream_t st) {
  const Operands o{Ahi, Alo, ldpa, p.M, B.hi, B.lo, B.ldp, p.N};
  return launch<F16X3_PRESPLIT>(o, p, st);
}

// split A once (stream-ordered scratch, same bytes as the fp32 original), then the TMA -> wgmma kernel on the planes
static int gemm_presplit(const float* A, int lda, const BOperand& B, const Params& p, cudaStream_t st) {
  const int M = p.M, K = p.K, ldpa = round_up(K, 8);
  __half* planes = nullptr;
  keep_stream_scratch_cached();
  MMX_CHECK_CUDA(cudaMallocAsync((void**)&planes, (size_t)2 * M * ldpa * sizeof(__half), st));
  __half *Ahi = planes, *Alo = planes + (size_t)M * ldpa;
  const long long total = (long long)M * ((K + 3) / 4);
  const int grid = (int)((total + 255) / 256 < (long long)sm_count() * 8 ? (total + 255) / 256 : (long long)sm_count() * 8);
  split_a_planes_kernel<<<grid, 256, 0, st>>>(A, lda, Ahi, Alo, ldpa, M, K, p.ep.a_act);
  MMX_LAUNCH_CHECK();
  const int rc = gemm_planes(Ahi, Alo, ldpa, B, p, st);
  cudaFreeAsync(planes, st);
  return rc;
}

}  // namespace wg

// get (bn < 0) / set the forced tile width; 0 = automatic
int gemm_tc_tile_n(int bn) {
  static std::atomic<int> forced{-1};
  if (forced.load() < 0) { const char* e = getenv("MMX_TC_BN"); const int v = e ? atoi(e) : 0; forced.store(v == 128 || v == 144 || v == 160 ? v : 0); }
  if (bn == 0 || bn == 128 || bn == 144 || bn == 160) forced.store(bn);
  return forced.load();
}

int gemm_tc_available() {
  // per device (a process may drive several GPUs); -1 = not probed yet
  static std::atomic<int> avail[MMX_MAX_DEVICES];
  static std::atomic<bool> init{false};
  static std::mutex mu;
  if (!init.load(std::memory_order_acquire)) {
    std::lock_guard<std::mutex> lk(mu);
    if (!init.load()) {
      for (auto& a : avail) a.store(-1);
      init.store(true, std::memory_order_release);
    }
  }
  const int dev = current_device();
  int a = avail[dev].load(std::memory_order_acquire);
  if (a >= 0) return a;
  std::lock_guard<std::mutex> lk(mu);
  a = 0;
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, dev) == cudaSuccess && prop.major == 9 && prop.minor == 0) {   // wgmma: sm_90a only
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) == cudaSuccess && fn != nullptr) {
      wg::g_encode = (PFN_cuTensorMapEncodeTiled_v12000)fn;
      a = 1;
    }
  }
  avail[dev].store(a, std::memory_order_release);
  return a;
}

// Which problems go to the tensor-core kernel.  Deliberately independent of M, so that a sample computed alone
// and the same sample inside a batch take the same arithmetic path (bitwise-equal maps, sharded == single GPU).
bool gemm_tc_shape_ok(const float* A, int lda, const float* Bt, int ldb, float* C, int ldc, int N, int K,
                      const GemmEpilogue& ep) {
  if (!gemm_tc_available()) return false;
  if (N < 128 || K < 64 || (N % 4) || (lda % 4) || (ldb % 4) || (ldc % 4)) return false;   // K itself is free: TMA zero-fills the tail
  if (!aligned16(A) || !aligned16(Bt) || !aligned16(C)) return false;
  if ((ep.bias && !aligned16(ep.bias)) || (ep.pre && (!aligned16(ep.pre) || ep.ldpre % 4)) ||
      (ep.residual && (!aligned16(ep.residual) || ep.ldres % 4)) || (ep.C_act && !aligned16(ep.C_act)))
    return false;
  return true;
}

int gemm_nt_tc(const float* A, int lda, const float* Bt, int ldb, float* C, int ldc, int M, int N, int K,
               const GemmEpilogue& ep, cudaStream_t st) {
  if (M == 0 || N == 0) return 0;
  const wg::Params p{M, N, K, ldc, C, ep};
  const wg::Operands o{A, nullptr, lda, M, Bt, nullptr, ldb, N};
  return wg::launch<wg::TF32X3>(o, p, st);
}

// `batch` independent products in ONE launch: C[b] = A[b] Bt[b]^T (+ residual[b]); A[b] starts rows_a rows after A[b-1] (same
// lda), Bt[b] rows_b rows after Bt[b-1]; a tile's operand boxes may run into the next sample's rows - those rows / columns
// of the product are never stored.
int gemm_nt_tc_batched(const float* A, int lda, int rows_a, const float* Bt, int ldb, int rows_b, float* C, int ldc, long long stride_c,
                       long long stride_res, int M, int N, int K, int batch, const GemmEpilogue& ep, cudaStream_t st) {
  if (M == 0 || N == 0 || batch == 0) return 0;
  MMX_REQUIRE(ep.m_dev == nullptr && ep.pre == nullptr && ep.C_act == nullptr && ep.bias == nullptr, "batched GEMM: residual epilogue only");
  wg::Params p{M, N, K, ldc, C, ep};
  p.batch = batch; p.rows_a = rows_a; p.rows_b = rows_b; p.stride_c = stride_c; p.stride_res = stride_res;
  const wg::Operands o{A, nullptr, lda, (batch - 1) * rows_a + M, Bt, nullptr, ldb, (batch - 1) * rows_b + N};
  return wg::launch<wg::TF32X3>(o, p, st);
}

int pack_f16x3_ld(int K) { return round_up(K, 8); }
size_t pack_f16x3_bytes(int N, int K) { return (size_t)2 * N * pack_f16x3_ld(K) * sizeof(uint16_t); }

int pack_f16x3(const float* W, int ldw, int N, int K, void* packed, cudaStream_t st) {
  if (N == 0 || K == 0) return 0;
  MMX_REQUIRE(aligned16(packed), "packed operand must be 16-byte aligned");
  const int ldp = pack_f16x3_ld(K);
  __half* hi = reinterpret_cast<__half*>(packed);
  __half* lo = hi + (size_t)N * ldp;
  const long long total = (long long)N * ldp;
  const long long cap = (long long)sm_count() * 8;
  const int grid = (int)((total + 255) / 256 < cap ? (total + 255) / 256 : cap);
  wg::pack_f16x3_kernel<<<grid, 256, 0, st>>>(W, ldw, hi, lo, ldp, N, K);
  MMX_LAUNCH_CHECK();
  return 0;
}

BOperand packed_operand(const float* W, int ldw, const void* packed, int N, int K) {
  BOperand B;
  B.w = W; B.ldw = ldw;
  if (packed) {
    B.ldp = pack_f16x3_ld(K);
    B.hi = reinterpret_cast<const uint16_t*>(packed);
    B.lo = B.hi + (size_t)N * B.ldp;
  }
  return B;
}

// The part of the fp16x3 rule that does not depend on how A arrives (fp32, or already split into planes): the packed B,
// the output, the epilogue operands and the tile minimums.
static bool f16x3_b_epilogue_ok(const BOperand& B, float* C, int ldc, int N, int K, const GemmEpilogue& ep) {
  if (!gemm_tc_available() || !B.hi || !B.lo) return false;
  if (N < 128 || K < 64 || (N % 4) || (B.ldp % 8) || (ldc % 4)) return false;   // K itself is free: TMA zero-fills the tail
  if (!aligned16(B.hi) || !aligned16(B.lo) || !aligned16(C)) return false;
  if ((ep.bias && !aligned16(ep.bias)) || (ep.pre && (!aligned16(ep.pre) || ep.ldpre % 4)) ||
      (ep.residual && (!aligned16(ep.residual) || ep.ldres % 4)) || (ep.C_act && !aligned16(ep.C_act)))
    return false;
  return true;
}

// Which problems go to the fp16x3 kernels.  Independent of M (a sample alone and inside a batch take the same arithmetic path).
bool gemm_f16x3_shape_ok(const float* A, int lda, const BOperand& B, float* C, int ldc, int N, int K, const GemmEpilogue& ep) {
  return (lda % 4) == 0 && aligned16(A) && f16x3_b_epilogue_ok(B, C, ldc, N, K, ep);
}

int gemm_nt_f16x3(const float* A, int lda, const BOperand& B, float* C, int ldc, int M, int N, int K, const GemmEpilogue& ep,
                  cudaStream_t st, bool presplit) {
  if (M == 0 || N == 0) return 0;
  const wg::Params p{M, N, K, ldc, C, ep};
  if (presplit) return wg::gemm_presplit(A, lda, B, p, st);
  const wg::Operands o{A, nullptr, lda, M, B.hi, B.lo, B.ldp, N};
  return wg::launch<wg::F16X3>(o, p, st);
}

bool gemm_f16x3_planes_ok(int ldpa, const BOperand& B, float* C, int ldc, int N, int K, const GemmEpilogue& ep) {
  return (ldpa % 8) == 0 && ldpa >= K && f16x3_b_epilogue_ok(B, C, ldc, N, K, ep);
}

int gemm_nt_f16x3_planes(const uint16_t* Ahi, const uint16_t* Alo, int ldpa, const BOperand& B, float* C, int ldc, int M, int N,
                         int K, const GemmEpilogue& ep, cudaStream_t st) {
  if (M == 0 || N == 0) return 0;
  const wg::Params p{M, N, K, ldc, C, ep};
  return wg::gemm_planes(reinterpret_cast<const __half*>(Ahi), reinterpret_cast<const __half*>(Alo), ldpa, B, p, st);
}

}  // namespace mmx
