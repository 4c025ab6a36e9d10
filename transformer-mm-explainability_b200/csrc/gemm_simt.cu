// fp32 FFMA GEMM  C[M,N] = A[M,K] * Bt[N,K]^T  with fused epilogues.  This is the accuracy/bisecting reference
// backend (and the fallback for shapes the wgmma kernels do not take: tiny test configs, K % 32 != 0).
// 128x128x16 CTA tile, 256 threads, 8x8 register tile per thread, double-buffered shared memory.
#include "mmx_common.cuh"
#include "gemm.cuh"

namespace mmx {

constexpr int TM = 128, TN = 128, TK = 16;

template <bool VEC>
__global__ void __launch_bounds__(256) gemm_nt_simt_kernel(const float* __restrict__ A, int lda,
                                                           const float* __restrict__ Bt, int ldb, float* __restrict__ C,
                                                           int ldc, int M, int N, int K, GemmEpilogue ep) {
  __shared__ __align__(16) float As[2][TK][TM + 4];
  __shared__ __align__(16) float Bs[2][TK][TN + 4];
  const int tid = threadIdx.x;
  if (ep.m_dev) M = min(M, __ldg(ep.m_dev));
  const int m0 = blockIdx.y * TM, n0 = blockIdx.x * TN;
  if (m0 >= M) return;
  const int tx = tid & 15, ty = tid >> 4;
  // loader mapping: each thread moves two float4 of A and two of Bt per k-tile
  const int lrow = tid >> 2, lk = (tid & 3) * 4;
  float4 ra[2], rb[2];
  auto load_global = [&](int k0) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int r = lrow + i * 64;
      const int gk = k0 + lk;
      ra[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      rb[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (VEC) {
        if (m0 + r < M && gk < K) ra[i] = *reinterpret_cast<const float4*>(A + (long long)(m0 + r) * lda + gk);
        if (n0 + r < N && gk < K) rb[i] = *reinterpret_cast<const float4*>(Bt + (long long)(n0 + r) * ldb + gk);
      } else {   // arbitrary K / leading dims / alignment (e.g. the 3129-way LXMERT answer head)
        if (m0 + r < M) {
          const float* p = A + (long long)(m0 + r) * lda + gk;
          if (gk + 0 < K) ra[i].x = p[0];
          if (gk + 1 < K) ra[i].y = p[1];
          if (gk + 2 < K) ra[i].z = p[2];
          if (gk + 3 < K) ra[i].w = p[3];
        }
        if (n0 + r < N) {
          const float* p = Bt + (long long)(n0 + r) * ldb + gk;
          if (gk + 0 < K) rb[i].x = p[0];
          if (gk + 1 < K) rb[i].y = p[1];
          if (gk + 2 < K) rb[i].z = p[2];
          if (gk + 3 < K) rb[i].w = p[3];
        }
      }
    }
  };
  auto store_smem = [&](int buf) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int r = lrow + i * 64;
      As[buf][lk + 0][r] = ra[i].x; As[buf][lk + 1][r] = ra[i].y; As[buf][lk + 2][r] = ra[i].z; As[buf][lk + 3][r] = ra[i].w;
      Bs[buf][lk + 0][r] = rb[i].x; Bs[buf][lk + 1][r] = rb[i].y; Bs[buf][lk + 2][r] = rb[i].z; Bs[buf][lk + 3][r] = rb[i].w;
    }
  };
  float acc[8][8] = {};
  load_global(0);
  store_smem(0);
  __syncthreads();
  const int nk = cdiv(K, TK);
  for (int kt = 0; kt < nk; ++kt) {
    const int buf = kt & 1;
    if (kt + 1 < nk) load_global((kt + 1) * TK);
#pragma unroll
    for (int k = 0; k < TK; ++k) {
      const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][k][ty * 4]);
      const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][k][64 + ty * 4]);
      const float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 4]);
      const float4 b1 = *reinterpret_cast<const float4*>(&Bs[buf][k][64 + tx * 4]);
      const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if (kt + 1 < nk) {
      store_smem(buf ^ 1);
      __syncthreads();
    }
  }
  // epilogue
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int gm = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + i - 4);
    if (gm >= M) continue;
#pragma unroll
    for (int jh = 0; jh < 2; ++jh) {
      const int gn0 = n0 + jh * 64 + tx * 4;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int gn = gn0 + j;
        if (gn >= N) continue;
        float v = acc[i][jh * 4 + j];
        if (ep.bias) v += ep.bias[gn];
        if (ep.pre) v *= act_bwd(ep.pre[(long long)gm * ep.ldpre + gn], ep.act);
        if (ep.residual) v += ep.residual[(long long)gm * ep.ldres + gn];
        if (ep.C_act != C) C[(long long)gm * ldc + gn] = v;
        if (ep.C_act) ep.C_act[(long long)gm * ldc + gn] = act_fwd(v, ep.act);
      }
    }
  }
}

int gemm_nt_simt(const float* A, int lda, const float* Bt, int ldb, float* C, int ldc, int M, int N, int K,
                 const GemmEpilogue& ep, cudaStream_t st) {
  if (M == 0 || N == 0) return 0;
  dim3 grid(cdiv(N, TN), cdiv(M, TM));
  const bool vec = K % 4 == 0 && lda % 4 == 0 && ldb % 4 == 0 && aligned16(A) && aligned16(Bt);
  if (vec) gemm_nt_simt_kernel<true><<<grid, 256, 0, st>>>(A, lda, Bt, ldb, C, ldc, M, N, K, ep);
  else gemm_nt_simt_kernel<false><<<grid, 256, 0, st>>>(A, lda, Bt, ldb, C, ldc, M, N, K, ep);
  MMX_LAUNCH_CHECK();
  return 0;
}

}  // namespace mmx
