// GEMM backends shared declarations.
#pragma once
#include "mmx_common.cuh"

namespace mmx {

// In place: C may be the very matrix pre or residual is (same base and row stride; each element is read, then written,
// by one thread).  Operands that overlap C in any other way are not supported.
struct GemmEpilogue {
  const float* bias = nullptr;      // [N]: added first
  const float* pre = nullptr;       // [M,N]: multiply by act'(pre)  (dgrad through an activation)
  int ldpre = 0;
  const float* residual = nullptr;  // [M,N]: added last
  int ldres = 0;
  float* C_act = nullptr;           // [M,N] (row stride ldc): also store act(C); C_act == C stores act(C) only
  int act = MMX_ACT_NONE;
  const int* m_dev = nullptr;       // optional device-resident row count (<= M): M becomes an upper bound (ragged batches)
  // Not an epilogue: the product takes act(A) for A.  Only the fp16x3 pre-split path (backend 3) applies it, in its split
  // pass; gemm_nt_b fails on any other path (gemm_a_act_ok says in advance).
  int a_act = MMX_ACT_NONE;
};

// A K-major GEMM "B" operand [N,K]: the fp32 matrix and, for static weights, its fp16 hi / lo planes
// (hi = fp16(w), lo = fp16((w - hi) * 2048), row stride ldp elements; see gemm_wgmma.cu).  hi == nullptr: not packed.
struct BOperand {
  const float* w = nullptr;
  int ldw = 0;
  const uint16_t* hi = nullptr;
  const uint16_t* lo = nullptr;
  int ldp = 0;
};

// C[M,N] = A[M,K] * Bt[N,K]^T, both operands K-major.
int gemm_nt_simt(const float* A, int lda, const float* Bt, int ldb, float* C, int ldc, int M, int N, int K,
                 const GemmEpilogue& ep, cudaStream_t st);

// Backend dispatch: wgmma 3xTF32 when the backend is enabled and the shape qualifies (the rule depends on N, K and
// alignment only - never on M - so one sample alone and inside a batch take the same arithmetic path), else fp32 FFMA.
int gemm_nt(const float* A, int lda, const float* Bt, int ldb, float* C, int ldc, int M, int N, int K,
            const GemmEpilogue& ep, cudaStream_t st);

// Same product with a (possibly packed) B operand: backend 2 runs the fp16x3 tensor-core kernel when B carries its
// hi / lo planes and the shape qualifies; everything else goes through gemm_nt's rule.
int gemm_nt_b(const float* A, int lda, const BOperand& B, float* C, int ldc, int M, int N, int K, const GemmEpilogue& ep,
              cudaStream_t st);
// Whether gemm_nt_b takes this product with ep.a_act set (backend 3 and a shape its fp16x3 kernel accepts).
bool gemm_a_act_ok(const float* A, int lda, const BOperand& B, float* C, int ldc, int N, int K, const GemmEpilogue& ep);

// fp16x3 backends (gemm_wgmma.cu)
size_t pack_f16x3_bytes(int N, int K);                 // bytes of one packed operand (hi plane then lo plane)
int pack_f16x3_ld(int K);                              // row stride (elements) of the planes
int pack_f16x3(const float* W, int ldw, int N, int K, void* packed, cudaStream_t st);
BOperand packed_operand(const float* W, int ldw, const void* packed, int N, int K);
bool gemm_f16x3_shape_ok(const float* A, int lda, const BOperand& B, float* C, int ldc, int N, int K, const GemmEpilogue& ep);
// presplit = true: backend 3 (A split into fp16 planes by a separate pass before the kernel)
int gemm_nt_f16x3(const float* A, int lda, const BOperand& B, float* C, int ldc, int M, int N, int K, const GemmEpilogue& ep,
                  cudaStream_t st, bool presplit = false);
// The backend-3 kernel on an A that is already split into fp16 hi / lo' planes [M, ldpa] (the conv gather writes them):
// same kernel and arithmetic as gemm_nt_f16x3(presplit = true) after its split pass.  The planes must be 16-byte aligned
// (the stream-ordered scratch they live in is); gemm_f16x3_planes_ok checks everything else.
bool gemm_f16x3_planes_ok(int ldpa, const BOperand& B, float* C, int ldc, int N, int K, const GemmEpilogue& ep);
int gemm_nt_f16x3_planes(const uint16_t* Ahi, const uint16_t* Alo, int ldpa, const BOperand& B, float* C, int ldc, int M, int N,
                         int K, const GemmEpilogue& ep, cudaStream_t st);
// gemm_nt_f16x3_planes inside the mmx_profile_gemm window (gemm_dispatch.cu)
int gemm_nt_planes(const uint16_t* Ahi, const uint16_t* Alo, int ldpa, const BOperand& B, float* C, int ldc, int M, int N, int K,
                   const GemmEpilogue& ep, cudaStream_t st);

int gemm_tc_available();
int gemm_tc_tile_n(int bn);   // forced tensor-core tile width: bn < 0 reads it, 0 = automatic, 128/144/160 force

// Tensor-core product for the relevancy updates (no bias / activation): C = residual + A * Bt^T with N possibly not a
// multiple of 4 as long as every row stride covers round_up(N, 4) columns (the pad columns receive zeros).  Returns
// taken = false when the shapes / alignment / backend do not qualify.
// Batched over `batch` samples in ONE launch: A[b] / Bt[b] start rows_a / rows_b rows after the previous sample (same leading
// dimension), residual / C advance by stride_res / stride_c elements.
int gemm_nt_tc_rule(const float* A, int lda, long long rows_a, const float* Bt, int ldb, long long rows_b, const float* residual,
                    int ldres, long long stride_res, float* C, int ldc, long long stride_c, int M, int N, int K, int batch,
                    cudaStream_t st, bool* taken);
int gemm_backend();

}  // namespace mmx
