// Relevancy rule kernels: rule 5 (Hadamard / clamp / head-mean), rules 6/7/10/11 (batched R updates),
// eq. 8-9 (row normalisation) and the rollout baseline.  See include/mmx.h for the reference lines replaced.
#include "mmx_common.cuh"
#include "gemm.cuh"
#include <math_constants.h>
#include <cstdlib>

namespace mmx {

// ---------------------------------------------------------------------------------------------------------
// Rule 5.  HBM-bound: reads 2*B*H*P floats, writes B*P.  Each thread owns one 128-bit column of the [T*S] plane
// and walks the H head planes, so the head reduction stays in registers (no cross-lane traffic needed) while a
// warp's loads stay fully coalesced (32 lanes x 16 B contiguous per head plane).
// ---------------------------------------------------------------------------------------------------------
template <int UNROLL>
__global__ void __launch_bounds__(256) avg_heads_vec4_kernel(const float* __restrict__ A, const float* __restrict__ G,
                                                             float* __restrict__ out, long long items, int PV, int H,
                                                             float inv_h) {
  // items = B * PV, PV = plane size in float4
  const long long plane = (long long)PV * 4;
  for (long long it = (long long)blockIdx.x * blockDim.x + threadIdx.x; it < items;
       it += (long long)gridDim.x * blockDim.x) {
    const long long b = it / PV;
    const int i = (int)(it - b * PV);
    const float* a = A + (b * H) * plane + 4LL * i;
    const float* g = G + (b * H) * plane + 4LL * i;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    int h = 0;
    for (; h + UNROLL <= H; h += UNROLL) {
      float4 av[UNROLL], gv[UNROLL];
#pragma unroll
      for (int u = 0; u < UNROLL; ++u) {
        av[u] = ld_stream4(a + (h + u) * plane);
        gv[u] = ld_stream4(g + (h + u) * plane);
      }
#pragma unroll
      for (int u = 0; u < UNROLL; ++u) {
        acc.x += relu_nan(av[u].x * gv[u].x);
        acc.y += relu_nan(av[u].y * gv[u].y);
        acc.z += relu_nan(av[u].z * gv[u].z);
        acc.w += relu_nan(av[u].w * gv[u].w);
      }
    }
    for (; h < H; ++h) {
      float4 av = ld_stream4(a + h * plane), gv = ld_stream4(g + h * plane);
      acc.x += relu_nan(av.x * gv.x);
      acc.y += relu_nan(av.y * gv.y);
      acc.z += relu_nan(av.z * gv.z);
      acc.w += relu_nan(av.w * gv.w);
    }
    acc.x *= inv_h; acc.y *= inv_h; acc.z *= inv_h; acc.w *= inv_h;
    *reinterpret_cast<float4*>(out + b * plane + 4LL * i) = acc;
  }
}

// attn-GradCAM baseline (DETR/modules/ExplanationGenerator.py:275-280): gbar[b,h] = mean_{t,s} dA[b,h,t,s], then
// out[b,t,s] = relu((1/H) sum_h A[b,h,t,s] * gbar[b,h]).  The plane sum runs in double: at DETR's long planes
// (T = S = 2500) each thread adds ~24k terms, and a signed gradient's mean can nearly cancel.
__global__ void __launch_bounds__(256) plane_mean_kernel(const float* __restrict__ G, float* __restrict__ gbar, int T, int S,
                                                         int ld) {
  __shared__ double red[8];
  const float* g = G + (long long)blockIdx.x * T * ld;
  double acc = 0.0;
  for (int e = threadIdx.x; e < T * S; e += blockDim.x) acc += (double)g[(long long)(e / S) * ld + e % S];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += red[w];
    gbar[blockIdx.x] = (float)(t / ((double)T * S));
  }
}
__global__ void __launch_bounds__(256) gradcam_kernel(const float* __restrict__ A, const float* __restrict__ gbar,
                                                      float* __restrict__ out, int B, int H, int T, int S, int ld_in,
                                                      int ld_out) {
  const long long items = (long long)B * T * S;
  const long long plane = (long long)T * ld_in;
  for (long long it = (long long)blockIdx.x * blockDim.x + threadIdx.x; it < items;
       it += (long long)gridDim.x * blockDim.x) {
    const int s = (int)(it % S);
    const long long r = it / S;
    const int t = (int)(r % T);
    const long long b = r / T;
    const long long off = (b * H) * plane + (long long)t * ld_in + s;
    float acc = 0.f;
    for (int h = 0; h < H; ++h) acc = fmaf(A[off + h * plane], gbar[b * H + h], acc);
    out[(b * T + t) * ld_out + s] = relu_nan(acc / (float)H);
  }
}

// generic strided / unaligned form (32-bit coalesced loads)
__global__ void __launch_bounds__(256) avg_heads_scalar_kernel(const float* __restrict__ A, const float* __restrict__ G,
                                                               float* __restrict__ out, int B, int H, int T, int S,
                                                               int ld_in, int ld_out, float inv_h) {
  const long long items = (long long)B * T * S;
  const long long plane = (long long)T * ld_in;
  for (long long it = (long long)blockIdx.x * blockDim.x + threadIdx.x; it < items;
       it += (long long)gridDim.x * blockDim.x) {
    const int s = (int)(it % S);
    const long long r = it / S;
    const int t = (int)(r % T);
    const long long b = r / T;
    const long long off = (b * H) * plane + (long long)t * ld_in + s;
    float acc = 0.f;
#pragma unroll 4
    for (int h = 0; h < H; ++h) acc += relu_nan(ld_stream1(A + off + h * plane) * ld_stream1(G + off + h * plane));
    out[(b * T + t) * ld_out + s] = acc * inv_h;
  }
}

// ---------------------------------------------------------------------------------------------------------
// Batched fp32 GEMM  C[b] = add[b] + op(A[b]) * B[b]   (64x64x16 tiles, 4x4 per thread).
// Used for every R update; sizes are small and arbitrary (S in {20,36,50,77,100,197,577,625,850}).
// ---------------------------------------------------------------------------------------------------------
constexpr int BT = 64, BKK = 16;

template <bool TRANS_A>
__global__ void __launch_bounds__(256) bmm_add_kernel(const float* __restrict__ A, int lda, long long sA,
                                                      const float* __restrict__ Bm, int ldb, long long sB,
                                                      const float* __restrict__ add, int ldadd, long long sAdd,
                                                      float* __restrict__ C, int ldc, long long sC, int M, int N,
                                                      int K, int nan_to_zero) {
  __shared__ float As[BKK][BT + 4];
  __shared__ float Bs[BKK][BT + 4];
  const int b = blockIdx.z;
  A += b * sA; Bm += b * sB; C += b * sC;
  if (add) add += b * sAdd;
  const int m0 = blockIdx.y * BT, n0 = blockIdx.x * BT;
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  float acc[4][4] = {};
  for (int k0 = 0; k0 < K; k0 += BKK) {
    // A tile -> As[k][m]
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int e = tid + i * 256;
      int m, k;
      if (TRANS_A) { k = e / BT; m = e % BT; } else { m = e / BKK; k = e % BKK; }
      const int gm = m0 + m, gk = k0 + k;
      float v = 0.f;
      if (gm < M && gk < K) v = TRANS_A ? A[(long long)gk * lda + gm] : A[(long long)gm * lda + gk];
      As[k][m] = v;
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int e = tid + i * 256;
      const int k = e / BT, n = e % BT;
      const int gk = k0 + k, gn = n0 + n;
      Bs[k][n] = (gk < K && gn < N) ? Bm[(long long)gk * ldb + gn] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < BKK; ++k) {
      const float4 av = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
      const float4 bv = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
      const float a[4] = {av.x, av.y, av.z, av.w}, bb[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], bb[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int gm = m0 + ty * 4 + i;
    if (gm >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int gn = n0 + tx * 4 + j;
      if (gn >= N) continue;
      float v = acc[i][j];
      if (nan_to_zero && isnan(v)) v = 0.f;
      if (add) v += add[(long long)gm * ldadd + gn];
      C[(long long)gm * ldc + gn] = v;
    }
  }
}

// eq. 8-9, one warp per row;  mode 0: (R-I)/rowsum(R-I)+I   mode 1 (rollout): (R+I)/rowsum(R+I)
__global__ void __launch_bounds__(256) row_normalize_kernel(const float* __restrict__ R, float* __restrict__ out, int ld,
                                                            int ldo, int rows_total, int S, int mode,
                                                            float* __restrict__ min_diag) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (min_diag != nullptr && blockIdx.x == 0) {
    // diag(R-I) minimum over the whole batch (the reference asserts it is >= 0 on the host)
    __shared__ float red[8];
    float m = CUDART_INF_F;
    for (int r = threadIdx.x; r < rows_total; r += blockDim.x) m = min_nan(m, R[(long long)r * ld + (r % S)] - 1.f);
    for (int o = 16; o > 0; o >>= 1) m = min_nan(m, __shfl_xor_sync(0xffffffffu, m, o));
    if (lane == 0) red[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int w = 1; w < (int)(blockDim.x >> 5); ++w) m = min_nan(m, red[w]);
      *min_diag = m;
    }
  }
  if (warp >= rows_total) return;
  const int i = warp % S;
  const float* r = R + (long long)warp * ld;
  float* o = out + (long long)warp * ldo;
  const float d = (mode == 0) ? -1.f : 1.f;
  float sum = 0.f;
  for (int s = lane; s < S; s += 32) sum += r[s] + (s == i ? d : 0.f);
  sum = warp_sum(sum);
  for (int s = lane; s < S; s += 32) {
    const float v = r[s] + (s == i ? d : 0.f);
    o[s] = (mode == 0) ? v / sum + (s == i ? 1.f : 0.f) : v / sum;
  }
}

__global__ void __launch_bounds__(256) copy2d_kernel(const float* __restrict__ src, int lds, float* __restrict__ dst,
                                                     int ldd, long long rows, int cols, int nan_to_zero, float add_diag,
                                                     int diag_period) {
  const long long n = rows * cols;
  for (long long it = (long long)blockIdx.x * blockDim.x + threadIdx.x; it < n; it += (long long)gridDim.x * blockDim.x) {
    const long long r = it / cols;
    const int c = (int)(it - r * cols);
    float v = src[r * lds + c];
    if (nan_to_zero && isnan(v)) v = 0.f;
    if (diag_period > 0 && (int)(r % diag_period) == c) v += add_diag;
    dst[r * ldd + c] = v;
  }
}

static int grid_for(long long items, int block = 256) {
  long long g = (items + block - 1) / block;
  long long cap = (long long)sm_count() * 8;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}

int bmm_add(const float* A, int lda, long long sA, int transA, const float* Bm, int ldb, long long sB, const float* add,
            int ldadd, long long sAdd, float* C, int ldc, long long sC, int batch, int M, int N, int K, int nan_to_zero,
            cudaStream_t st) {
  MMX_REQUIRE(batch >= 0 && M >= 0 && N >= 0 && K >= 0, "negative dims");
  if (batch == 0 || M == 0 || N == 0) return 0;
  for (int b0 = 0; b0 < batch; b0 += 65535) {
    const int nb = batch - b0 < 65535 ? batch - b0 : 65535;
    dim3 grid(cdiv(N, BT), cdiv(M, BT), nb);
    const float* addp = add ? add + b0 * sAdd : nullptr;
    if (transA)
      bmm_add_kernel<true><<<grid, 256, 0, st>>>(A + b0 * sA, lda, sA, Bm + b0 * sB, ldb, sB, addp, ldadd, sAdd,
                                                 C + b0 * sC, ldc, sC, M, N, K, nan_to_zero);
    else
      bmm_add_kernel<false><<<grid, 256, 0, st>>>(A + b0 * sA, lda, sA, Bm + b0 * sB, ldb, sB, addp, ldadd, sAdd,
                                                  C + b0 * sC, ldc, sC, M, N, K, nan_to_zero);
    MMX_LAUNCH_CHECK();
  }
  return 0;
}

// out[b][n][k] = in[b][k][n] for n < N, k < K, zero in the pads (out is [batch][Np][Kp] dense): the K-major "B"
// operand of the tensor-core product  R + Abar * R  (the GEMM kernel takes both operands K-major).
__global__ void __launch_bounds__(256) transpose_pad_kernel(const float* __restrict__ in, int ld_in, long long s_in,
                                                            float* __restrict__ out, int K, int N, int Kp, int Np) {
  __shared__ float t[32][33];
  const int b = blockIdx.z;
  in += b * s_in;
  out += (long long)b * Np * Kp;
  const int n0 = blockIdx.x * 32, k0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int i = ty; i < 32; i += 8) {
    const int k = k0 + i, n = n0 + tx;
    t[i][tx] = (k < K && n < N) ? in[(long long)k * ld_in + n] : 0.f;
  }
  __syncthreads();
  for (int i = ty; i < 32; i += 8) {
    const int n = n0 + i, k = k0 + tx;
    if (n < Np && k < Kp) out[(long long)n * Kp + k] = t[tx][i];
  }
}

// Rules 6/7 on the tensor cores:  C[b] = R[b] + Abar[b] * R[b]   for S >= 128 (DETR 625-850, ViT-B/16 197, ViT-L 577).
// One transpose of every sample's R into a K-major scratch, then ONE batched wgmma 3xTF32 GEMM launch (tile -> sample,
// row block, column block) with the "+R" fused as the residual epilogue.  Small S (CLIP 50/77, LXMERT 20/36) stays on the FFMA kernel: a 128x128 tensor tile would be mostly padding.
int self_update_tc(const float* Abar, int ld_a, const float* R, float* R_out, int ld, int B, int S, int Q, cudaStream_t st,
                   bool* taken) {
  *taken = false;
  if (gemm_backend() < 1 || S < 128 || Q < 128 || (ld_a % 4) || (ld % 4) || ld < round_up(Q, 4) || !aligned16(Abar) ||
      !aligned16(R) || !aligned16(R_out))
    return 0;
  keep_stream_scratch_cached();
  const int Kp = round_up(S, 4), Np = round_up(Q, 4);
  float* Rt = nullptr;
  MMX_CHECK_CUDA(cudaMallocAsync((void**)&Rt, (size_t)B * Np * Kp * sizeof(float), st));
  dim3 grid(cdiv(Np, 32), cdiv(Kp, 32), B);
  transpose_pad_kernel<<<grid, 256, 0, st>>>(R, ld, (long long)S * ld, Rt, S, Q, Kp, Np);
  count_launch();
  // ONE launch for all samples: tile -> (sample, row block, column block); Abar[b] is S rows after Abar[b-1], Rt[b] Np rows
  bool ok = false;
  int rc = gemm_nt_tc_rule(Abar, ld_a, S, Rt, Kp, Np, R, ld, (long long)S * ld, R_out, ld, (long long)S * ld, S, Q, S, B, st, &ok);
  if (rc == 0 && !ok) { rc = 3; set_error("tensor-core rule GEMM rejected a shape it was offered"); }
  cudaFreeAsync(Rt, st);
  *taken = rc == 0;
  return rc;
}

int avg_heads(const float* A, const float* dA, float* Abar, int B, int H, int T, int S, int ld_in, int ld_out,
              cudaStream_t st) {
  MMX_REQUIRE(B >= 0 && H > 0 && T >= 0 && S >= 0 && ld_in >= S && ld_out >= S, "bad dims");
  if (B == 0 || T == 0 || S == 0) return 0;
  const float inv_h = 1.f / (float)H;
  const long long P = (long long)T * S;
  if (ld_in == S && ld_out == S && (P % 4) == 0 && aligned16(A) && aligned16(dA) && aligned16(Abar)) {
    const int PV = (int)(P / 4);
    const long long items = (long long)B * PV;
    // heads in flight per thread (2 x UNROLL 128-bit loads) and CTAs per SM (profiles/rule5_sweep.py sweeps both)
    static int unroll = -1, per_sm = -1;
    if (unroll < 0) {
      const char* e = getenv("MMX_AVG_UNROLL");
      unroll = e ? atoi(e) : 8;
      e = getenv("MMX_AVG_CTAS_PER_SM");
      per_sm = e ? atoi(e) : 16;
    }
    long long g = (items + 255) / 256, cap = (long long)sm_count() * per_sm;
    const int grid = (int)(g > cap ? cap : g);
    switch (unroll) {
      case 2: avg_heads_vec4_kernel<2><<<grid, 256, 0, st>>>(A, dA, Abar, items, PV, H, inv_h); break;
      case 6: avg_heads_vec4_kernel<6><<<grid, 256, 0, st>>>(A, dA, Abar, items, PV, H, inv_h); break;
      case 8: avg_heads_vec4_kernel<8><<<grid, 256, 0, st>>>(A, dA, Abar, items, PV, H, inv_h); break;
      case 12: avg_heads_vec4_kernel<12><<<grid, 256, 0, st>>>(A, dA, Abar, items, PV, H, inv_h); break;
      default: avg_heads_vec4_kernel<4><<<grid, 256, 0, st>>>(A, dA, Abar, items, PV, H, inv_h); break;
    }
  } else {
    avg_heads_scalar_kernel<<<grid_for((long long)B * T * S), 256, 0, st>>>(A, dA, Abar, B, H, T, S, ld_in, ld_out, inv_h);
  }
  MMX_LAUNCH_CHECK();
  return 0;
}

int handle_residual(const float* R, float* out, int ld, int ldo, int B, int S, int mode, float* min_diag, cudaStream_t st) {
  if (B == 0 || S == 0) return 0;
  const int rows = B * S;
  row_normalize_kernel<<<cdiv(rows, 8), 256, 0, st>>>(R, out, ld, ldo, rows, S, mode, min_diag);
  MMX_LAUNCH_CHECK();
  return 0;
}

int copy2d(const float* src, int lds, float* dst, int ldd, long long rows, int cols, int nan_to_zero, cudaStream_t st) {
  if (rows == 0 || cols == 0) return 0;
  copy2d_kernel<<<grid_for(rows * cols), 256, 0, st>>>(src, lds, dst, ldd, rows, cols, nan_to_zero, 0.f, 0);
  MMX_LAUNCH_CHECK();
  return 0;
}

// min and max of one map over a 256-thread CTA, as torch's cam.min() / cam.max(): one NaN makes both NaN (fminf / fmaxf
// would skip it).  Every thread gets the result.
__device__ __forceinline__ void block_minmax_nan(float& mn, float& mx) {
  __shared__ float smn[8], smx[8];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    mn = min_nan(mn, __shfl_xor_sync(0xffffffffu, mn, o));
    mx = max_nan(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  }
  if ((threadIdx.x & 31) == 0) { smn[threadIdx.x >> 5] = mn; smx[threadIdx.x >> 5] = mx; }
  __syncthreads();
  mn = smn[0]; mx = smx[0];
#pragma unroll
  for (int w = 1; w < 8; ++w) { mn = min_nan(mn, smn[w]); mx = max_nan(mx, smx[w]); }
}

// y = (x - min(x)) / (max(x) - min(x)) over each of B contiguous maps of n floats (one CTA per map).  A constant map
// gives 0/0 = NaN and a map holding a NaN gives NaN everywhere, exactly as the reference expression does.
__global__ void __launch_bounds__(256) minmax_normalize_kernel(const float* __restrict__ X, float* __restrict__ Y, long long n) {
  const float* x = X + (long long)blockIdx.x * n;
  float* y = Y + (long long)blockIdx.x * n;
  float mn = INFINITY, mx = -INFINITY;
  for (long long i = threadIdx.x; i < n; i += blockDim.x) { const float v = x[i]; mn = min_nan(mn, v); mx = max_nan(mx, v); }
  block_minmax_nan(mn, mx);
  const float d = mx - mn;
  for (long long i = threadIdx.x; i < n; i += blockDim.x) y[i] = (x[i] - mn) / d;
}

// Otsu mask of one map per CTA (DETR/mask_generator.py:115-121): min-max -> *255 -> uint8 (truncation) -> 256-bin
// histogram (shared-memory integer atomics: order-independent) -> OpenCV's getThreshVal_Otsu_8u scan in double by one
// thread (256 steps, the same operation order as the CPU library so the threshold is bit-identical) -> 0 / 255.
__global__ void __launch_bounds__(256) otsu_mask_kernel(const float* __restrict__ X, float* __restrict__ M,
                                                       int* __restrict__ thresholds, int n) {
  const float* x = X + (long long)blockIdx.x * n;
  float* m = M + (long long)blockIdx.x * n;
  __shared__ int hist[256];
  __shared__ int s_thr;
  float mn = INFINITY, mx = -INFINITY;
  for (int i = threadIdx.x; i < n; i += blockDim.x) { const float v = x[i]; mn = min_nan(mn, v); mx = max_nan(mx, v); }
  hist[threadIdx.x] = 0;
  block_minmax_nan(mn, mx);                                  // its barrier also orders the histogram clear
  const float d = mx - mn;
  auto quant = [&](float v) -> int {                       // ((v - min) / (max - min)) * 255 in fp32, then astype(uint8)
    const float q = __fmul_rn(__fdiv_rn(__fsub_rn(v, mn), d), 255.f);
    return q >= 0.f ? (int)q & 255 : 0;                      // NaN (constant map, or a NaN anywhere in it) -> 0, as numpy's
  };                                                         // cast gives on x86: every pixel lands in bin 0, mask all 0
  for (int i = threadIdx.x; i < n; i += blockDim.x) atomicAdd(&hist[quant(x[i])], 1);
  __syncthreads();
  if (threadIdx.x == 0) {
    const double scale = 1.0 / (double)n;
    double mu = 0.0;
    for (int i = 0; i < 256; ++i) mu += (double)i * (double)hist[i];
    mu *= scale;
    double mu1 = 0.0, q1 = 0.0, max_sigma = 0.0;
    int max_val = 0;
    const double eps = 1.1920928955078125e-07;              // FLT_EPSILON
    for (int i = 0; i < 256; ++i) {
      const double p_i = (double)hist[i] * scale;
      mu1 = __dmul_rn(mu1, q1);
      q1 += p_i;
      const double q2 = 1.0 - q1;
      if (fmin(q1, q2) < eps || fmax(q1, q2) > 1.0 - eps) continue;
      mu1 = __ddiv_rn(__dadd_rn(mu1, __dmul_rn((double)i, p_i)), q1);
      const double mu2 = __ddiv_rn(__dsub_rn(mu, __dmul_rn(q1, mu1)), q2);
      const double diff = __dsub_rn(mu1, mu2);
      const double sigma = __dmul_rn(__dmul_rn(__dmul_rn(q1, q2), diff), diff);
      if (sigma > max_sigma) { max_sigma = sigma; max_val = i; }
    }
    s_thr = max_val;
    if (thresholds) thresholds[blockIdx.x] = max_val;
  }
  __syncthreads();
  const int thr = s_thr;
  for (int i = threadIdx.x; i < n; i += blockDim.x) m[i] = quant(x[i]) > thr ? 255.f : 0.f;
}

// Top-k selection by rank for the perturbation drivers (lxmert/lxmert/perturbation.py:110-113,160-172: `cam.topk(k)` then
// gather): keep[i] = 1 if fewer than k elements beat element i (greater score, or equal score and lower index; a NaN
// beats every number, as torch.topk ranks it, and NaNs among themselves follow the index rule), pos[i] = number of kept
// elements before i in INDEX order (the compacted position after the reference's `sorted`), or -1.  The ranks are a
// permutation of 0..n-1, so exactly clamp(k, 0, n) elements are kept.  One CTA per row; n <= 4096.
__global__ void __launch_bounds__(256) topk_select_kernel(const float* __restrict__ scores, int n, const int* __restrict__ k,
                                                         int* __restrict__ keep, int* __restrict__ pos) {
  extern __shared__ float sh[];
  float* sv = sh;
  int* sk = reinterpret_cast<int*>(sh + n);
  const float* x = scores + (long long)blockIdx.x * n;
  const int kk = k[blockIdx.x];
  for (int i = threadIdx.x; i < n; i += blockDim.x) sv[i] = x[i];
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const float v = sv[i];
    const bool v_nan = v != v;
    int rank = 0;
    for (int j = 0; j < n; ++j) {
      const float u = sv[j];
      rank += (u != u) ? (!v_nan || j < i) : (!v_nan && (u > v || (u == v && j < i)));
    }
    sk[i] = rank < kk;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    int before = 0;
    for (int j = 0; j < i; ++j) before += sk[j];
    keep[(long long)blockIdx.x * n + i] = sk[i];
    pos[(long long)blockIdx.x * n + i] = sk[i] ? before : -1;
  }
}

}  // namespace mmx

using namespace mmx;

extern "C" {

int mmx_avg_heads(const float* A, const float* dA, float* Abar, int B, int H, int T, int S, int ld_in, int ld_out,
                  void* stream) {
  return avg_heads(A, dA, Abar, B, H, T, S, ld_in, ld_out, (cudaStream_t)stream);
}

int mmx_attn_gradcam(const float* A, const float* dA, float* out, float* gbar, int B, int H, int T, int S, int ld_in,
                     int ld_out, void* stream) {
  MMX_REQUIRE(B >= 0 && H > 0 && ld_in >= S && ld_out >= S && gbar != nullptr, "bad arguments");
  if (B == 0 || T == 0 || S == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  plane_mean_kernel<<<B * H, 256, 0, st>>>(dA, gbar, T, S, ld_in);
  MMX_LAUNCH_CHECK();
  gradcam_kernel<<<grid_for((long long)B * T * S), 256, 0, st>>>(A, gbar, out, B, H, T, S, ld_in, ld_out);
  MMX_LAUNCH_CHECK();
  return 0;
}

int mmx_bmm_add(const float* A, int lda, long long strideA, int transA, const float* Bm, int ldb, long long strideB,
                const float* add, int ldadd, long long strideAdd, float* C, int ldc, long long strideC, int batch, int M,
                int N, int K, void* stream) {
  return bmm_add(A, lda, strideA, transA, Bm, ldb, strideB, add, ldadd, strideAdd, C, ldc, strideC, batch, M, N, K, 0,
                 (cudaStream_t)stream);
}

int mmx_self_update(const float* Abar, int ld_a, const float* R_ss, float* R_ss_out, int ld_ss, const float* R_sq,
                    float* R_sq_out, int ld_sq, int B, int S, int Q, void* stream) {
  MMX_REQUIRE(R_ss != R_ss_out && (R_sq == nullptr || R_sq != R_sq_out), "outputs may not alias inputs");
  cudaStream_t st = (cudaStream_t)stream;
  bool tc = false;
  MMX_TRY(self_update_tc(Abar, ld_a, R_ss, R_ss_out, ld_ss, B, S, S, st, &tc));
  if (!tc)
    MMX_TRY(bmm_add(Abar, ld_a, (long long)S * ld_a, 0, R_ss, ld_ss, (long long)S * ld_ss, R_ss, ld_ss,
                    (long long)S * ld_ss, R_ss_out, ld_ss, (long long)S * ld_ss, B, S, S, S, 0, st));
  if (R_sq != nullptr && Q > 0) {
    tc = false;
    MMX_TRY(self_update_tc(Abar, ld_a, R_sq, R_sq_out, ld_sq, B, S, Q, st, &tc));
    if (!tc)
      MMX_TRY(bmm_add(Abar, ld_a, (long long)S * ld_a, 0, R_sq, ld_sq, (long long)S * ld_sq, R_sq, ld_sq,
                      (long long)S * ld_sq, R_sq_out, ld_sq, (long long)S * ld_sq, B, S, Q, S, 0, st));
  }
  return 0;
}

int mmx_handle_residual(const float* R, float* out, int ld, int B, int S, float* min_diag, void* stream) {
  return handle_residual(R, out, ld, ld, B, S, 0, min_diag, (cudaStream_t)stream);
}

size_t mmx_mm_update_workspace(int B, int T, int S) {
  return sizeof(float) * (size_t)B * ((size_t)T * T + (size_t)S * S + (size_t)T * S);
}

int mmx_mm_update(const float* R_ss, int ld_ss, const float* R_qq, int ld_qq, const float* R_qs, int ld_qs,
                  const float* Abar_sq, int ld_a, float* R_sq_add, int ld_sq_add, float* R_ss_add, int ld_ss_add, int B,
                  int T, int S, int flags, void* workspace, float* min_diag, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  MMX_REQUIRE(workspace != nullptr, "workspace required");
  float* ws_ss = (float*)workspace;
  float* ws_qq = ws_ss + (size_t)B * T * T;
  float* ws_t = ws_qq + (size_t)B * S * S;
  const int nan0 = (flags & MMX_MM_NAN_TO_ZERO) ? 1 : 0;
  if (flags & MMX_MM_SELF_IN_10) {
    const float *Xs = R_ss, *Xq = R_qq;
    int lxs = ld_ss, lxq = ld_qq;
    if (flags & MMX_MM_NORMALIZE) {
      MMX_TRY(handle_residual(R_ss, ws_ss, ld_ss, T, B, T, 0, min_diag, st));
      MMX_TRY(handle_residual(R_qq, ws_qq, ld_qq, S, B, S, 0, min_diag ? min_diag + 1 : nullptr, st));
      Xs = ws_ss; lxs = T; Xq = ws_qq; lxq = S;
    }
    // tmp[T,S] = Abar_sq * Rn_qq ;  add = Rn_ss^T * tmp
    MMX_TRY(bmm_add(Abar_sq, ld_a, (long long)T * ld_a, 0, Xq, lxq, (long long)S * lxq, nullptr, 0, 0, ws_t, S,
                    (long long)T * S, B, T, S, S, 0, st));
    MMX_TRY(bmm_add(Xs, lxs, (long long)T * lxs, 1, ws_t, S, (long long)T * S, nullptr, 0, 0, R_sq_add, ld_sq_add,
                    (long long)T * ld_sq_add, B, T, S, T, nan0, st));
  } else {
    // the reference normalises (and asserts diag(R - I) >= 0) before it discards the product
    // (DETR/modules/ExplanationGenerator.py:36-41), so the assert's operand is still produced
    if ((flags & MMX_MM_NORMALIZE) && min_diag) {
      MMX_TRY(handle_residual(R_ss, ws_ss, ld_ss, T, B, T, 0, min_diag, st));
      MMX_TRY(handle_residual(R_qq, ws_qq, ld_qq, S, B, S, 0, min_diag + 1, st));
    }
    // R_sq_addition = cam_sq (a copy; NaN->0 still applies for DETR)
    for (int b = 0; b < B; ++b)
      MMX_TRY(copy2d(Abar_sq + (size_t)b * T * ld_a, ld_a, R_sq_add + (size_t)b * T * ld_sq_add, ld_sq_add, T, S, nan0, st));
  }
  if (R_qs != nullptr && R_ss_add != nullptr)
    MMX_TRY(bmm_add(Abar_sq, ld_a, (long long)T * ld_a, 0, R_qs, ld_qs, (long long)S * ld_qs, nullptr, 0, 0, R_ss_add,
                    ld_ss_add, (long long)T * ld_ss_add, B, T, T, S, 0, st));
  return 0;
}

int mmx_rollout(const float* mats, int L, int B, int S, int start_layer, int normalize, float* out, float* workspace,
                void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  MMX_REQUIRE(L > 0 && start_layer >= 0 && start_layer < L, "start_layer out of range");
  const long long msz = (long long)B * S * S;
  float* cur = workspace;          // normalised layer matrix
  float* alt = workspace + msz;    // ping-pong partner of `out`
  // choose buffers so that the final product lands in `out`
  const int steps = L - 1 - start_layer;
  float* joint = (steps % 2 == 0) ? out : alt;
  auto prep = [&](int l, float* dst) -> int {
    if (normalize) return handle_residual(mats + l * msz, dst, S, S, B, S, 1, nullptr, st);
    copy2d_kernel<<<grid_for(msz), 256, 0, st>>>(mats + l * msz, S, dst, S, (long long)B * S, S, 0, 1.f, S);
    MMX_LAUNCH_CHECK();
    return 0;
  };
  MMX_TRY(prep(start_layer, joint));
  for (int l = start_layer + 1; l < L; ++l) {
    MMX_TRY(prep(l, cur));
    float* nxt = (joint == out) ? alt : out;
    MMX_TRY(bmm_add(cur, S, (long long)S * S, 0, joint, S, (long long)S * S, nullptr, 0, 0, nxt, S, (long long)S * S, B, S,
                    S, S, 0, st));
    joint = nxt;
  }
  return 0;
}

int mmx_minmax_normalize(const float* X, float* Y, int B, long long n, void* stream) {
  MMX_REQUIRE(B >= 0 && n > 0, "empty map");
  if (B == 0) return 0;
  minmax_normalize_kernel<<<B, 256, 0, (cudaStream_t)stream>>>(X, Y, n);
  MMX_LAUNCH_CHECK();
  return 0;
}

int mmx_otsu_masks(const float* cams, float* masks, int* thresholds, int B, int n, void* stream) {
  MMX_REQUIRE(B >= 0 && n > 0, "empty map");
  if (B == 0) return 0;
  otsu_mask_kernel<<<B, 256, 0, (cudaStream_t)stream>>>(cams, masks, thresholds, n);
  MMX_LAUNCH_CHECK();
  return 0;
}

int mmx_topk_select(const float* scores, const int* k, int* keep, int* pos, int B, int n, void* stream) {
  MMX_REQUIRE(B >= 0 && n > 0 && n <= 4096, "row length must be in 1..4096");
  if (B == 0) return 0;
  topk_select_kernel<<<B, 256, (size_t)n * 8, (cudaStream_t)stream>>>(scores, n, k, keep, pos);
  MMX_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
