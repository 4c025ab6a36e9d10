/*
 * mmx.h - C ABI of libmmx.so, the H100-native (sm_90a) gradient-weighted attention-relevancy engine.
 *
 * The reference (hila-chefer/Transformer-MM-Explainability) is 100 % Python/PyTorch and defines NO FFI or
 * plugin layer (SURVEY.md §8b): its boundary is a set of Python call signatures.  This header is therefore
 * the contract a maintainer of the reference would bind (ctypes stub shown in INTEGRATION.md); each entry
 * point cites the reference function (file:line under the reference tree) whose arithmetic it replaces.
 *
 * Conventions
 *   - plain C: raw DEVICE pointers (fp32 unless said otherwise), explicit sizes / leading dimensions, a
 *     cudaStream_t passed as void* (NULL = legacy default stream).  No torch / C++ types.
 *   - every function returns 0 on success, non-zero on error; mmx_last_error() returns the text (thread-local).
 *   - the caller allocates all outputs; kernels never allocate.  The only hidden allocations are the engine
 *     objects (mmx_clip_create), which own their weight arena and activation workspace.
 *   - "ld*" arguments are row strides in ELEMENTS; "plane" strides are computed as rows*ld.
 *   - nothing here falls back to the CPU: if no sm_90 device is present the calls fail.
 */
#ifndef MMX_H_
#define MMX_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MMX_VERSION 1

const char* mmx_last_error(void);
int mmx_version(void);
/* Number of kernels this library has launched since load (all streams); the bench reports it as gpu_launches. */
uint64_t mmx_launch_count(void);
/* Selects the GEMM backend for the transformer linears: 0 = fp32 FFMA (bisecting reference), 1 = wgmma 3xTF32
 * (raw fp32 operands split on the SM), 2 = wgmma fp16x3 (three f16 passes over fp16 hi / lo planes, the weights
 * pre-split once with mmx_pack_weight, the activations split inside the GEMM kernel; linears whose weight is not packed
 * run as backend 1), 3 = the same arithmetic with the activations split into planes by a separate pass before the
 * kernel (default when available: faster on H100, see DESIGN.md §4.1).
 * All four are fp32-faithful (<= 2e-5 of max|C| against fp64).  Env MMX_GEMM_BACKEND overrides the default.
 * Returns the backend in effect. */
int mmx_set_gemm_backend(int backend);
/* The backend in effect.  The LRP sweeps (use_lrp=True) switch to backend 0 for their forward, backward and relprop and
 * restore this value afterwards: relprop divides by activations and sums that nearly cancel, which amplifies the 1e-6
 * rounding of the tensor-core splits by several orders of magnitude (measured: tests/test_lrp_gpu.py). */
int mmx_get_gemm_backend(void);
/* Tile width of the tensor-core backends: 0 = automatic (the width in {128, 144, 160} whose tile count best fills whole
 * waves of SMs), or one of 128 / 144 / 160 to force it (profiling and the bit-equality test: the width never changes a
 * result bit).  Env MMX_TC_BN sets the initial value.  Returns the value in effect. */
int mmx_set_gemm_tile_n(int bn);
/* Per-launch CUDA-event timing of the transformer GEMMs (the dominant kernel): enable=1 opens a window, enable=0
 * closes it; the report synchronises the device and returns the summed launch durations, the algorithmic FLOPs
 * (2*M*N*K per launch) and the launch count of the window.  Used by bench.py for the roofline line. */
int mmx_profile_gemm(int enable);
int mmx_profile_gemm_report(double* total_ms, double* total_flops, int* launches);
/* Profiling aid: while set, the attention forward kernel writes CTA 0's clock64 timeline of its 7 phase boundaries into
 * device_buf[4096 ..] (4112 int64 in all); NULL switches it off.  profiles/attn_trace.py. */
int mmx_gemm_trace(long long* device_buf);
/* Device-to-device copy on `stream` (used by the test taps; avoids a second CUDA runtime binding on the host side). */
int mmx_memcpy_d2d(void* dst, const void* src, size_t bytes, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * Rule kernels (SURVEY.md §8a rows a5-a9)
 * ------------------------------------------------------------------------------------------------------- */

/* Rule 5:  Abar[b,t,s] = (1/H) * sum_h max(dA[b,h,t,s] * A[b,h,t,s], 0).
 * Replaces avg_heads (DETR/modules/ExplanationGenerator.py:19-24; lxmert/lxmert/src/ExplanationGenerator.py:18-23)
 * and the inline batched form of CLIP_explainability.ipynb:176-181 (head index b*H+h).
 * A, dA: [B,H,T,S] with row stride ld_in; Abar: [B,T,S] with row stride ld_out.  HBM-bound. */
int mmx_avg_heads(const float* A, const float* dA, float* Abar, int B, int H, int T, int S,
                  int ld_in, int ld_out, void* stream);

/* attn-GradCAM baseline:  out[b,t,s] = relu( (1/H) sum_h A[b,h,t,s] * mean_{t',s'} dA[b,h,t',s'] ).
 * Replaces gradcam() (DETR/modules/ExplanationGenerator.py:275-280; lxmert/lxmert/src/ExplanationGenerator.py:542-547).
 * gbar: device scratch of B*H floats; each plane mean is summed in double, so it is the fp32 rounding of the exact mean
 * even when a signed gradient nearly cancels over a long plane (T = S = 2500). */
int mmx_attn_gradcam(const float* A, const float* dA, float* out, float* gbar, int B, int H, int T, int S, int ld_in,
                     int ld_out, void* stream);

/* Rules 6+7:  R_ss_out = R_ss + Abar*R_ss ;  R_sq_out = R_sq + Abar*R_sq  (both from the PRE-update state).
 * Replaces apply_self_attention_rules + the caller's "+=" (DETR/modules/ExplanationGenerator.py:27-30,118,
 * 127-129) and "R = R + torch.bmm(cam, R)" (CLIP_explainability.ipynb:182,205).
 * Abar [B,S,S] (ld_a), R_ss [B,S,S] (ld_ss), R_sq [B,S,Q] (ld_sq) or NULL.  Outputs may not alias inputs.
 * For S >= 128 (and Q >= 128) with row strides that are multiples of 4 covering round_up(cols, 4) zero-padded columns,
 * the product runs on the tensor cores (wgmma 3xTF32, "+R" fused as the epilogue residual); smaller or unaligned
 * problems use the fp32 FFMA kernel. */
int mmx_self_update(const float* Abar, int ld_a, const float* R_ss, float* R_ss_out, int ld_ss,
                    const float* R_sq, float* R_sq_out, int ld_sq, int B, int S, int Q, void* stream);

/* Eq. 8-9:  out = (R - I) / rowsum(R - I) + I.  Replaces handle_residual
 * (DETR/modules/ExplanationGenerator.py:46-53).  The reference asserts diag(R-I) >= 0 on the host; here the
 * minimum diagonal entry of R-I over the batch is written to *min_diag (device float, may be NULL) so the
 * caller can raise the same AssertionError without a sync inside the kernel. */
int mmx_handle_residual(const float* R, float* out, int ld, int B, int S, float* min_diag, void* stream);

#define MMX_MM_NORMALIZE     1   /* apply_normalization=True  */
#define MMX_MM_SELF_IN_10    2   /* apply_self_in_rule_10=True */
#define MMX_MM_NAN_TO_ZERO   4   /* DETR's R_sq_addition[isnan]=0 (DETR/modules/ExplanationGenerator.py:42) */

/* Rules 10+11.  R_sq_add = Rn_ss^T * (Abar_sq * Rn_qq)   (Rn = handle_residual(R) when MMX_MM_NORMALIZE, else R;
 * R_sq_add = Abar_sq when !MMX_MM_SELF_IN_10);  R_ss_add = Abar_sq * R_qs  (only when R_qs != NULL).
 * Replaces apply_mm_attention_rules (DETR/modules/ExplanationGenerator.py:33-43 - returns R_sq_add only, with
 * NaN->0; lxmert/lxmert/src/ExplanationGenerator.py:32-42 - returns (R_sq_add, R_ss_add), no NaN guard).
 * Shapes per sample: R_ss [T,T], R_qq [S,S], Abar_sq [T,S], R_qs [S,T]; outputs R_sq_add [T,S], R_ss_add [T,T].
 * workspace: device scratch of mmx_mm_update_workspace(B,T,S) bytes.  min_diag: 2 device floats (ss, qq) or NULL. */
size_t mmx_mm_update_workspace(int B, int T, int S);
int mmx_mm_update(const float* R_ss, int ld_ss, const float* R_qq, int ld_qq, const float* R_qs, int ld_qs,
                  const float* Abar_sq, int ld_a, float* R_sq_add, int ld_sq_add, float* R_ss_add, int ld_ss_add,
                  int B, int T, int S, int flags, void* workspace, float* min_diag, void* stream);

/* The whole rule-6 chain of one tower in ONE launch: R = I, then R <- R + Abar[l] R for l = 0 .. L-1, with R resident in
 * shared memory and the products on the tensor cores (mma.sync 3xTF32).  Replaces the per-block `R = R + torch.bmm(cam, R)`
 * loop (CLIP_explainability.ipynb:169-183; ViT ipynb:1193-1199; VisualBERT ExplanationGenerator.py:84-93).
 * Abar: [L][B][S][ld] (layer_stride elements between layers, S*ld between samples, ld % 4 == 0, pad columns zero);
 * R_out: [B][S][ld_out].  S <= 128 (larger S: mmx_self_update per layer, which runs on the wgmma GEMM). */
int mmx_self_chain(const float* Abar, long long layer_stride, int ld, float* R_out, int ld_out, int B, int S, int L,
                   void* stream);

/* Rollout baseline: prod_l rownorm(mats[l] + I), l = start_layer .. L-1, later layers multiplied on the left.
 * Replaces compute_rollout_attention (DETR/modules/ExplanationGenerator.py:5-16; normalize=0 gives the
 * VisualBERT variant, VisualBERT/mmf/models/transformers/backends/ExplanationGenerator.py:5-17).
 * mats: [L,B,S,S] contiguous (ld = S);  out: [B,S,S];  workspace: 2*B*S*S floats. */
int mmx_rollout(const float* mats, int L, int B, int S, int start_layer, int normalize, float* out,
                float* workspace, void* stream);

/* Min-max normalisation of B contiguous maps of n floats: Y = (X - min X) / (max X - min X) per map (in place allowed).
 * Replaces the `(cam - cam.min()) / (cam.max() - cam.min())` step of the attn-GradCAM / partial-LRP baselines
 * (VisualBERT/mmf/models/transformers/backends/ExplanationGenerator.py:122,203) and of the DETR mask generator
 * (DETR/mask_generator.py:115-121).  A constant map yields NaN, as in the reference.  min and max propagate NaN as
 * torch's cam.min() / cam.max() do: a map holding a NaN yields NaN everywhere. */
int mmx_minmax_normalize(const float* X, float* Y, int B, long long n, void* stream);

/* Otsu masks for B relevance maps of n floats (the step right after the path in the DETR segmentation driver):
 * masks[b] = 255 where uint8((cam - min) / (max - min) * 255) > otsu_threshold else 0, thresholds[b] (optional) = the
 * threshold.  Replaces DETR/mask_generator.py:115-121 (`cv2.threshold(..., THRESH_BINARY + THRESH_OTSU)` on the CPU with
 * a device->host->device round trip per query); bit-identical to OpenCV's getThreshVal_Otsu_8u.  A map holding a NaN
 * (or a constant map) normalises to NaN everywhere, which the uint8 cast turns into 0 as numpy does on x86: threshold 0,
 * mask all 0. */
int mmx_otsu_masks(const float* cams, float* masks, int* thresholds, int B, int n, void* stream);

/* Top-k selection for the perturbation drivers: for each of B rows of n scores, keep[b][i] = 1 for the k[b] highest
 * scores (ties: lower index first), pos[b][i] = rank of i among the kept elements in index order, -1 when dropped.
 * NaN ranks above every number, as in torch.topk (among NaNs the lower index first); exactly clamp(k[b], 0, n) elements
 * are kept.  n <= 4096.
 * Replaces `cam.topk(k)` + host-side `sorted(...)` + gather (lxmert/lxmert/perturbation.py:110-117,160-178). */
int mmx_topk_select(const float* scores, const int* k, int* keep, int* pos, int B, int n, void* stream);

/* Generic batched C[b] = beta_src[b] + op(A[b]) * B[b]  (fp32, used by the rule entry points above; exported
 * for the host-side generators).  transA: 0 = A is [M,K], 1 = A is stored [K,M].  add may be NULL. */
int mmx_bmm_add(const float* A, int lda, long long strideA, int transA, const float* Bm, int ldb, long long strideB,
                const float* add, int ldadd, long long strideAdd, float* C, int ldc, long long strideC,
                int batch, int M, int N, int K, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * Transformer primitives that produce A and dA (SURVEY.md §8a rows a2, a3, a11, a13).  Exported so the
 * host-side generators for DETR / LXMERT / ViT can be assembled from the same kernels as the CLIP engine.
 * ------------------------------------------------------------------------------------------------------- */

#define MMX_ACT_NONE       0
#define MMX_ACT_QUICKGELU  1   /* x*sigmoid(1.702x), CLIP/clip/model.py:162-164 */
#define MMX_ACT_GELU       2   /* exact erf GELU (timm ViT, LXMERT) */
#define MMX_ACT_RELU       3   /* DETR FFN, DETR/models/transformer.py:239; NaN propagates as in F.relu (relu(NaN) = NaN)
                                  and the derivative passes the gradient where pre is NaN (threshold_backward) */
#define MMX_ACT_TANH       4   /* LXMERT pooler, lxmert/lxmert/src/lxmert_lrp.py:868-884 */
#define MMX_ACT_MUL        5   /* not an activation: the `pre` operand of a GEMM epilogue multiplies the product itself
                                  (C = (A W^T) (.) pre), the `x * (S W)` step of Linear.relprop, DETR/modules/layers.py:421-423 */
#define MMX_ACT_SIGMOID    6   /* 1/(1+exp(-x)): DETR's box head, `self.bbox_embed(hs).sigmoid()` DETR/models/detr.py:73 */

/* C[M,N] = A[M,K] * W[N,K]^T (+ bias[N]) (+ residual[M,N]);  if act != NONE and C_act != NULL also writes
 * C_act = act(C); C_act == C stores act(C) only (a forward-only consumer that never needs the pre-activation).
 * F.linear of CLIP/clip/auxilary.py:77,255 and CLIP/clip/model.py:175-177. */
int mmx_linear(const float* A, int lda, const float* W, int ldw, const float* bias, const float* residual,
               int ldres, float* C, int ldc, float* C_act, int act, int M, int N, int K, void* stream);
/* dX[M,K] = (dY[M,N] * W[N,K]) (.) act'(pre[M,K])   given Wt = W^T stored [K,N]:  the dgrad of mmx_linear,
 * optionally continued through the activation that PRODUCED this linear's input (pre = that activation's
 * pre-activation; NULL = none).  The reference obtains it through torch.autograd (CLIP_explainability.ipynb:175). */
int mmx_linear_dgrad(const float* dY, int lddy, const float* Wt, int ldwt, const float* pre, int ldpre, int act,
                     float* dX, int lddx, int M, int N, int K, void* stream);

/* fp16x3 operand packing for STATIC weights (backend 2): packed holds the fp16 planes hi = fp16(w) and
 * lo = fp16((w - hi) * 2048), each [N, round_up(K, 8)], mmx_pack_weight_bytes(N, K) bytes in total (4 bytes per element,
 * like the fp32 original), 16-byte aligned device memory owned by the caller.  Re-pack after the weight changes.
 * mmx_linear_packed / mmx_linear_dgrad_packed are mmx_linear / mmx_linear_dgrad with the packed copy of the SAME matrix
 * (W for the forward, W^T for the dgrad) beside the fp32 pointer; packed == NULL is exactly the unpacked call.
 * Range: |x| <= 65504 for both operands (larger values produce inf / NaN, never a silently wrong number); magnitudes
 * below ~1e-5 keep an absolute precision of 3e-11 (scale tiny gradient streams by a power of two, see
 * mmx_attention_bwd_scaled). */
size_t mmx_pack_weight_bytes(int N, int K);
int mmx_pack_weight(const float* W, int ldw, int N, int K, void* packed, void* stream);
int mmx_linear_packed(const float* A, int lda, const float* W, int ldw, const void* packed, const float* bias,
                      const float* residual, int ldres, float* C, int ldc, float* C_act, int act, int M, int N, int K,
                      void* stream);
int mmx_linear_dgrad_packed(const float* dY, int lddy, const float* Wt, int ldwt, const void* packed_t, const float* pre,
                            int ldpre, int act, float* dX, int lddx, int M, int N, int K, void* stream);

/* The general form behind the four entry points above:  C = ((A[M,K] * Bt[N,K]^T + bias) (.) act'(pre)) + residual, and
 * C_act = act(C) when given.  bias / pre / residual / C_act / packed may be NULL.  With act = MMX_ACT_MUL the product is
 * multiplied by `pre` itself. */
int mmx_gemm_nt(const float* A, int lda, const float* Bt, int ldb, const void* packed, const float* bias, const float* pre,
                int ldpre, const float* residual, int ldres, float* C, int ldc, float* C_act, int act, int M, int N, int K,
                void* stream);

/* Small glue kernels for the host-side generators (DETR / LXMERT / ViT orchestration; row-major [rows, cols] with
 * row strides in elements).  They replace elementwise torch ops of the reference models (positional-embedding adds
 * DETR/models/transformer.py:236,378-390; residual adds; x[:,0] / embedding gathers). */
/* out = a + alpha*b  (out may alias a) */
int mmx_add(const float* a, int lda, const float* b, int ldb, float alpha, float* out, int ldo, long long rows, int cols,
            void* stream);
/* out[r,:] = src[row_map[r],:] */
int mmx_gather_rows(const float* src, int lds, const int32_t* row_map, float* out, int ldo, int rows, int cols, void* stream);
/* dst[row_map[r],:] += src[r,:]   (row_map entries must be distinct) */
int mmx_scatter_add_rows(const float* src, int lds, const int32_t* row_map, float* dst, int ldd, int rows, int cols,
                         void* stream);
/* dx = dy (.) act'(pre)  and  y = act(x) as standalone elementwise passes */
int mmx_act_bwd(const float* dy, int lddy, const float* pre, int ldpre, int act, float* dx, int lddx, long long rows, int cols,
                void* stream);
int mmx_act_fwd(const float* x, int ldx, int act, float* y, int ldy, long long rows, int cols, void* stream);
/* images [n,3,R,R] -> patches [n*(R/p)^2, 3*p*p] in conv-weight order (the conv1 of CLIP/clip/model.py:230 and of the
 * timm ViT patch embedding, as a GEMM operand) */
int mmx_im2col_patches(const float* images, float* patches, int n_images, int resolution, int patch, void* stream);

/* LayerNorm over the last dim (eps 1e-5), optional row gather: out row r reads x row row_map[r].
 * CLIP/clip/model.py:153-159.  mean/rstd ([rows]) are saved for the backward. */
int mmx_layernorm_fwd(const float* x, int ldx, const int* row_map, const float* gamma, const float* beta,
                      float* y, int ldy, float* mean, float* rstd, int rows, int D, float eps, void* stream);
/* dx[out_row] = (residual_grad ? residual_grad[out_row] : 0) + LN'(dy; x, mean, rstd, gamma);
 * out row = row_map ? row_map[r] : r (x is read at the same mapped row). */
int mmx_layernorm_bwd(const float* dy, int lddy, const float* x, int ldx, const int* row_map, const float* gamma,
                      const float* mean, const float* rstd, const float* residual_grad, int ldres, float* dx,
                      int lddx, int rows, int D, void* stream);

#define MMX_ATTN_CAUSAL        1   /* additive -inf above the diagonal, CLIP/clip/model.py:334-340 */
#define MMX_ATTN_SCALE_SCORES  2   /* scores/sqrt(d) after QK^T (lxmert_lrp.py:398-399); default: q scaled first
                                      (CLIP/clip/auxilary.py:153) */

/* A = softmax(scale * Q K^T + mask) staged to HBM, O = A V.   Q [B,T,H*hd] (ldq), K,V [B,S,H*hd] (ldk, ldv),
 * key_bias [B,S] additive or NULL, A [B,H,T,S] row stride ldA, O [B,T,H*hd] (ldo).
 * Replaces the bmm/softmax/bmm of CLIP/clip/auxilary.py:225-252, DETR/modules/layers.py:753-762,
 * lxmert/lxmert/src/lxmert_lrp.py:398-414, including the "save A" hook sites (:247-250 / :758 / :407).
 * hd in {16, 32, 64}; S up to 16384 keys.  Up to 1024 keys (when the score rows of a 32- or 64-query tile fit in shared
 * memory) one pass per query tile; longer rows run a two-pass kernel (row statistics, then normalised tiles), chosen by
 * shape alone.  Ragged batches take at most 1024 keys.  The products are 3xTF32 tensor-core
 * passes (error vs fp64 ~1e-6), the softmax is fp32.  A key_bias of -inf REMOVES the key (its probability is exactly 0,
 * the same bits a -10000 mask gives); a row whose keys are all removed gets A = 0 and O = 0 (softmax over an empty set). */
int mmx_attention_fwd(const float* Q, int ldq, const float* K, int ldk, const float* V, int ldv,
                      const float* key_bias, float* A, int ldA, float* O, int ldo,
                      int B, int H, int T, int S, int hd, float scale, int flags, void* stream);
/* Backward from dO: dA = dO V^T staged to HBM (the tensor the reference captures with register_hook,
 * CLIP/clip/auxilary.py:250), then dS = A (.) (dA - rowsum(dA (.) A)), dQ, dK, dV.  dQ/dK/dV may all be NULL
 * (stop after dA).  delta: scratch [B,H,T]. */
int mmx_attention_bwd(const float* dO, int lddo, const float* Q, int ldq, const float* K, int ldk,
                      const float* V, int ldv, const float* A, float* dA, int ldA, float* delta,
                      float* dQ, int lddq, float* dK, int lddk, float* dV, int lddv,
                      int B, int H, int T, int S, int hd, float scale, int flags, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * DETR backbone from images (SURVEY.md §8a rows a10, a11): the ResNet body, input_proj and the mask / sine position
 * embedding that DETR.forward runs before the transformer (DETR/models/detr.py:63-69, DETR/models/backbone.py:68-121).
 * Activations are NHWC matrices [B*H*W, C] (row = (b*H + y)*W + x) with a row stride in elements.
 * ------------------------------------------------------------------------------------------------------- */

/* out[B*Ho*Wo, Cout] = act(conv2d(x, W) + bias (+ residual)), Ho = (H + 2 pad - kh) / stride + 1 (same for Wo), zero
 * padding.  Replaces the Conv2d + FrozenBatchNorm2d (+ ReLU, + identity add) steps of torchvision's ResNet
 * (DETR/models/backbone.py:45-55,91-93) and DETR's input_proj (DETR/models/detr.py:44,69) once the BN affine is folded
 * into W and bias.  x is addressed through element strides (sN, sY, sX, sC) - an NCHW image and an NHWC activation with
 * any row stride are both valid inputs.  W: [Cout, kh*kw*C] in (ky, kx, c) order (row stride ldw), packed: its
 * mmx_pack_weight copy or NULL.  A 1x1 stride-1 conv over rows with unit channel stride is a plain mmx_gemm_nt; every
 * other conv gathers its [B*Ho*Wo, kh*kw*C] operand once (under backend 3 straight into the fp16 hi / lo planes the
 * GEMM loads, elsewhere as fp32) into stream-ordered scratch.  act: MMX_ACT_*; the pre-activation is not stored.
 * residual: [B*Ho*Wo, Cout] (row stride ldres) or NULL. */
int mmx_conv2d(const float* x, long long sN, long long sY, long long sX, long long sC, int B, int H, int W, int C,
               const float* Wr, int ldw, const void* packed, const float* bias, const float* residual, int ldres, float* out,
               int ldo, int Cout, int kh, int kw, int stride, int pad, int act, void* stream);
/* mmx_conv2d with a dilation (F.conv2d(dilation=dilation), DETR's DC5 layer4: torchvision's _make_layer(dilate=True),
 * DETR/models/backbone.py:88-90): tap (ky, kx) of output pixel (oy, ox) reads input pixel (oy stride - pad + ky dilation,
 * ox stride - pad + kx dilation), Ho = (H + 2 pad - dilation (kh - 1) - 1) / stride + 1 (same for Wo).  mmx_conv2d is
 * this entry point with dilation = 1. */
int mmx_conv2d_dilated(const float* x, long long sN, long long sY, long long sX, long long sC, int B, int H, int W, int C,
                       const float* Wr, int ldw, const void* packed, const float* bias, const float* residual, int ldres, float* out,
                       int ldo, int Cout, int kh, int kw, int stride, int pad, int dilation, int act, void* stream);
/* 3x3 / stride 2 / padding 1 max-pool over NHWC rows (padding acts as -inf, NaN propagates): torchvision ResNet's
 * maxpool (F.max_pool2d).  in: [B*H*W, C] (ldi), out: [B*Ho*Wo, C] (ldo), Ho = (H - 1) / 2 + 1. */
int mmx_maxpool2d_nhwc(const float* in, int ldi, float* out, int ldo, int B, int H, int W, int C, void* stream);
/* The padding mask at feature resolution and PositionEmbeddingSine(npf, temperature, normalize=True) of it, in one kernel.
 * mask: [B, Hi, Wi] bytes, non-zero = padding (NULL: no padding); it is sampled to [B, h, w] as F.interpolate(mode=
 * "nearest") does (DETR/models/backbone.py:78) and written to mask_out (bytes, may be NULL).  pos: [B*h*w, 2*npf] (row
 * stride ldpos, row = (b*h + y)*w + x, the layout the encoder reads), channels [0, npf) from y, [npf, 2 npf) from x,
 * sin / cos interleaved, in the reference's fp32 operation order (DETR/models/position_encoding.py:28-48).  h*w <= 16384;
 * one CTA per 32 positions of an image. */
int mmx_detr_position_sine(const uint8_t* mask, int B, int Hi, int Wi, int h, int w, int npf, float temperature, float* pos,
                           int ldpos, uint8_t* mask_out, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * DETR evaluation post-processing (the per-image body of DETR/engine.py:173-192, `--eval --masks`)
 * ------------------------------------------------------------------------------------------------------- */

/* PostProcess (DETR/models/detr.py:278-306) and the keep rule of MaskGenerator.get_panoptic (DETR/mask_generator.py:50-51)
 * in one kernel, one warp per (image, query) row.  logits: pred_logits [B*Q, C1] (row stride ld, C1 = classes + 1 >= 2);
 * prob = softmax(row); scores = max(prob[:C1-1]), labels = its index (int64; NaN wins, ties take the lower index, as
 * torch's max(-1)); keep = scores > keep_threshold (bytes; false for NaN).  A row holding a NaN or inf gives score NaN.
 * boxes: pred_boxes [B*Q, 4] (cx, cy, w, h); sizes: [B, 2] int64 (img_h, img_w), device memory;
 * boxes_out = box_cxcywh_to_xyxy(boxes) * (img_w, img_h, img_w, img_h), the same bits as torch.  Every output may be
 * NULL; boxes_out needs boxes and sizes. */
int mmx_detr_postprocess(const float* logits, int ld, int B, int Q, int C1, float keep_threshold, float* scores, int64_t* labels,
                         uint8_t* keep, const float* boxes, const int64_t* sizes, float* boxes_out, void* stream);
/* PostProcessSegm (DETR/models/segmentation.py:218-242) for a batch in one launch: F.interpolate(pred_masks, (max_h, max_w),
 * "bilinear", align_corners=False), sigmoid() > threshold, the crop [:img_h, :img_w] and F.interpolate(nearest) to
 * (oh, ow), as bytes 0 / 1.  pred_masks: [B, Q, h, w] fp32 (any values; h > 1); sizes, orig_sizes: HOST int arrays [B][2]
 * of (img_h, img_w) (target_sizes) and (oh, ow) (orig_target_sizes); (max_h, max_w) is the column max of sizes.
 * out: device bytes, image i's [Q, oh_i, ow_i] masks at offset sum_{j<i} Q oh_j ow_j.  Only the bilinear values the
 * nearest step reads are computed, with ATen's CUDA arithmetic, so the masks are the bits the reference's CUDA
 * interpolate + CPU resize gives.  B <= 64. */
int mmx_detr_segm_postprocess(const float* pred_masks, int B, int Q, int h, int w, const int* sizes, const int* orig_sizes,
                              float threshold, uint8_t* out, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * CLIP engine: the north-star path (SURVEY.md §8a rows a1-a4), one call = interpret() for a batch.
 * ------------------------------------------------------------------------------------------------------- */

typedef struct mmx_clip_config {
  /* constructor arguments of the reference CLIP (CLIP/clip/model.py:249-262), ViT image tower */
  int embed_dim, image_resolution, vision_layers, vision_width, vision_patch_size;
  int context_length, vocab_size, transformer_width, transformer_heads, transformer_layers;
} mmx_clip_config;

typedef struct mmx_clip mmx_clip;

/* max_batch = largest number of (image,text) pairs processed in one pass; larger batches are micro-batched. */
int mmx_clip_create(const mmx_clip_config* cfg, int max_batch, mmx_clip** out);
void mmx_clip_destroy(mmx_clip* h);
/* Load one tensor of the reference state_dict by its key (e.g. "visual.transformer.resblocks.0.attn.in_proj_weight",
 * CLIP/clip/model.py:405-442).  data: HOST fp32, numel elements. */
int mmx_clip_load_tensor(mmx_clip* h, const char* name, const float* data, size_t numel);
/* Checks that every tensor was loaded and builds the derived copies (transposed weights for the dgrad GEMMs). */
int mmx_clip_finalize(mmx_clip* h);

/* interpret() (CLIP_explainability.ipynb:151-208).  images: [n_images,3,R,R] fp32 with n_images == B or 1 (the
 * notebook's image.repeat, :153); tokens: [B,context] int32.  start_layer / start_layer_text as in the notebook
 * (-1 = last block only).  R_text: [B,ctx,ctx], R_image: [B,S_v-1].  *_device: all pointers are device memory,
 * work is enqueued on `stream`, after everything already enqueued there, and later work on `stream` is ordered after it
 * (NULL: the legacy default stream); the call does not wait for the results.  *_host: pointers
 * are host memory (pinned or pageable); copies happen inside the call, which returns after the results landed. */
int mmx_clip_interpret_device(mmx_clip* h, const float* images, int n_images, const int32_t* tokens, int B,
                              int start_layer, int start_layer_text, float* R_text, float* R_image, void* stream);
int mmx_clip_interpret_host(mmx_clip* h, const float* images, int n_images, const int32_t* tokens, int B,
                            int start_layer, int start_layer_text, float* R_text, float* R_image);

/* Measurement aid: serial != 0 puts both towers on ONE stream (results unchanged), so that per-launch CUDA-event times do
 * not overlap and the time of a kernel family is a true share of the step; 0 restores the two concurrent tower streams. */
int mmx_clip_set_serial(mmx_clip* h, int serial);

/* Test taps: device pointers into the engine workspace after the last interpret (valid for batch <= max_batch,
 * first micro-batch).  what: "A" / "dA" ([B,H,S,S]) / "Abar" ([B,S,S]) (tower 0 = vision, 1 = text, layer index),
 * "logits" ([B,B]); the residual stream "x" ([M,D], layer 0 .. L: x of layer l is the input of block l, layer L the tower
 * output), "xmid" ([M,D]), "qkv" ([M,3D]), "f" ([M,4D], fc1 before the activation) and "stats" ([4,M]: mean1, rstd1,
 * mean2, rstd2 of the block's two LayerNorms) of block `layer`; per tower, `layer` ignored: "feat", "featn", "dfeat"
 * ([B,E]: pooled features, their normalised copy, the seed gradient times gscale) and "gscale" ([B]).  M = B*S rows, except
 * for the ragged text tower: its rows are packed and M is the packed row count of the last call.
 * Writes the pointer, the dims (up to 4) and the row stride of the last dim. */
int mmx_clip_tap(mmx_clip* h, const char* what, int tower, int layer, const float** ptr, int dims[4], int* ld);

/* mmx_attention_bwd for a gradient stream that carries a per-sample power-of-two factor: dO (and hence delta, dQ, dK,
 * dV) are gscale[b] times the true gradients, the staged dA is divided by gscale[b] (exact) so that it is the tensor the
 * reference's hook sees.  gscale: [B] device floats, or NULL (= mmx_attention_bwd).  Used with the fp16x3 backend to keep
 * the dgrad operands inside fp16's exponent range. */
int mmx_attention_bwd_scaled(const float* dO, int lddo, const float* Q, int ldq, const float* K, int ldk,
                             const float* V, int ldv, const float* A, float* dA, int ldA, float* delta,
                             float* dQ, int lddq, float* dK, int lddk, float* dV, int lddv,
                             int B, int H, int T, int S, int hd, float scale, int flags, const float* gscale, void* stream);

/* Ragged self-attention, the CLIP text tower's packed rows: sample b owns rows offs[b] .. offs[b] + lens[b] - 1 of Q / K / V
 * / O (and of dO / dQ / dK / dV) and attends within them only (T = S = lens[b], 1 <= lens[b] <= T).  offs, lens: [B] device
 * ints (mmx_text_embed_packed writes them).  The staged A / dA planes stay dense [B,H,T,ldA]: rows and columns >= lens[b] are
 * written as 0.  Packed rows past sum(lens) are neither read nor written.  T <= 1024 and no key bias; otherwise as
 * mmx_attention_fwd / mmx_attention_bwd_scaled (gscale may be NULL; dQ / dK / dV all NULL stops after dA). */
int mmx_attention_fwd_ragged(const float* Q, int ldq, const float* K, int ldk, const float* V, int ldv, float* A, int ldA,
                             float* O, int ldo, const int* offs, const int* lens, int B, int H, int T, int hd, float scale,
                             int flags, void* stream);
int mmx_attention_bwd_ragged(const float* dO, int lddo, const float* Q, int ldq, const float* K, int ldk, const float* V,
                             int ldv, const float* A, float* dA, int ldA, float* delta, float* dQ, int lddq, float* dK,
                             int lddk, float* dV, int lddv, const int* offs, const int* lens, int B, int H, int T, int hd,
                             float scale, int flags, const float* gscale, void* stream);

/* The CLIP engine's token assembly and logit head as standalone calls (row-major, dense rows). */
/* Packed text embedding (CLIP/clip/model.py:350-352,360): lens[b] = 1 + the first argmax of tokens[b, 0:S] (the EOT; rows
 * after it cannot reach the pooled feature under the causal mask), offs = exclusive scan of lens, eot_row[b] = offs[b] +
 * lens[b] - 1, *total = sum(lens); x[offs[b] + s] = emb[tokens[b,s]] + pos[s] for s < lens[b] (token ids clamped to
 * [0, vocab)).  tokens: [B,S] int32, emb: [vocab,D], pos: [S,D], x: [B*S,D] (rows past *total untouched); all device. */
int mmx_text_embed_packed(const int32_t* tokens, const float* emb, const float* pos, float* x, int* offs, int* lens,
                          int* eot_row, int* total, int B, int S, int D, int vocab, void* stream);
/* Vision tokens with the ln_pre fused (CLIP/clip/model.py:233-235): x[b,0] = LN(cls + pos[0]), x[b,1+g] =
 * LN(patch_emb[(b % n_img)*(S-1) + g] + pos[1+g]).  patch_emb: [n_img*(S-1),D], pos: [S,D], x: [B*S,D]. */
int mmx_vision_tokens_lnpre(const float* patch_emb, int n_img, const float* cls, const float* pos, const float* gamma,
                            const float* beta, float* x, int B, int S, int D, float eps, void* stream);
/* Logit head and its analytic backward for y = sum_b logits_per_image[b,b] (CLIP/clip/model.py:368-374,
 * CLIP_explainability.ipynb:156-160), one warp per sample: fin / ftn = fi / |fi|, ft / |ft|; diag[b] = logit_scale_exp *
 * <fin_b, ftn_b> (diag may be NULL); dfi / dft = dy / d(fi, ft).  With gs_i / gs_t given, row b of dfi (dft) is multiplied
 * by the power of two gs_i[b] (gs_t[b]) that puts its max |.| in [16, 32) (1 when that max is 0 or not finite), and the
 * factors are written.  fi, ft, fin, ftn, dfi, dft: [B,E]. */
int mmx_clip_head(const float* fi, const float* ft, float logit_scale_exp, float* fin, float* ftn, float* dfi, float* dft,
                  float* diag, float* gs_i, float* gs_t, int B, int E, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * LRP (`relprop`) primitives: the second sweep behind use_lrp=True / generate_transformer_att / generate_partial_lrp
 * (SURVEY.md §8f-4).  The reference runs it through autograd (gradient x input per layer, DETR/modules/layers.py:38-66);
 * these are the same rules as direct kernels.  Matrices are row-major [B * rows_per_sample, cols] with row strides in
 * elements; one "sample" is what the reference treats as the whole tensor (it runs relprop with batch 1).
 * Whole-sample sums are carried as `partials`: mmx_lrp_partials_len() * k doubles per sample (k = 2: sum and abs-sum,
 * k = 3 inside mmx_lrp_add), reduced in a fixed order by the consumer, so results are deterministic.
 * ------------------------------------------------------------------------------------------------------- */
/* P = clamp(X, min=0), N = clamp(X, max=0): the positive / negative parts of Linear.relprop (layers.py:411-414) */
int mmx_lrp_split(const float* X, int ldx, float* P, float* N, int ld, long long rows, int cols, void* stream);
/* S = safe_divide(R, Z) (layers.py:11-14): R / (Z + 1e-9) (1e-9 when that is 0), and 0 where Z == 0 */
int mmx_lrp_safe_divide(const float* R, int ldr, const float* Z, int ldz, float* S, int lds, long long rows, int cols,
                        void* stream);
int mmx_lrp_partials_len(void);
/* partials[b][c] = {sum, sum of |x|} over chunk c of sample b (the `R.sum()`, `out.sum()`, `cam_v.min() == cam_v.max() == 0`
 * reductions of layers.py:430-432,786-799) */
int mmx_lrp_sums(const float* X, int ldx, int rows_per_sample, int cols, int B, double* partials, void* stream);
/* X[b] *= safe_divide(sum(num[b]), sum(den[b])): the renormalisation that ends DETR's Linear.relprop (layers.py:430-432) */
int mmx_lrp_renorm(float* X, int ldx, int rows_per_sample, int cols, int B, const double* num_partials,
                   const double* den_partials, void* stream);
/* Add.relprop (layers.py:194-221; lxmert/lxmert/src/layers.py Add): S = safe_divide(R, x0 + x1), a = x0 S, b = x1 S, each
 * rescaled to its share |sum a| : |sum b| of sum R.  b may be NULL.  workspace: 3 * partials_len doubles per sample. */
int mmx_lrp_add(const float* R, int ldr, const float* x0, int ld0, const float* x1, int ld1, float* a, int lda, float* b,
                int ldb, int rows_per_sample, int cols, int B, double* workspace, void* stream);
/* Clone.relprop (layers.py:252-270): out = X * sum_i safe_divide(R[i], X), i < n <= 8 (R: host array of device pointers).
 * With n = 1 it is also IndexSelect.relprop on the selected rows (layers.py:230-249). */
int mmx_lrp_clone(const float* X, int ldx, const float* const* R, const int* ldr, int n, float* out, int ldo, long long rows,
                  int cols, void* stream);
/* The all-zero-value case of MultiheadAttention.relprop (layers.py:786-799), decided per sample ON THE DEVICE: when the
 * value relevance is all zero after its projection but was not before, cam_q and cam_k are rescaled to share sum(cam). */
int mmx_lrp_zero_value_fix(float* cam_q, int ldq, int rows_q, float* cam_k, int ldk, int rows_k, int cols, int B,
                           const double* v_pre, const double* v_post, const double* q_sums, const double* k_sums,
                           const double* cam_sums, void* stream);
/* RelPropSimple through attn @ v (layers.py:776-781; lxmert_lrp.py:431-437): with Sv = safe_divide(R_o, O),
 * cam_A[b,h,i,j] = A (.) (Sv V^T) / 2 staged in A's [B,H,T,ldA] layout (pad columns zero) - this is `attn_cam` - and
 * cam_V[b*S+j, h*hd+d] = V (.) (A^T Sv) / 2.  R_o, O: [B*T, H*hd]; V: [B*S, H*hd]. */
int mmx_lrp_attn_pv(const float* R_o, int ldr, const float* O, int ldo, const float* A, int ldA, const float* V, int ldv,
                    float* cam_A, float* cam_V, int ldcv, int B, int H, int T, int S, int hd, void* stream);
/* RelPropSimple through q @ k^T (layers.py:783-785; lxmert_lrp.py:441-447): Z = zscale * Q K^T, S2 = safe_divide(cam1, Z),
 * cam_Q = (zscale Q) (.) (S2 K) / 2, cam_K = K (.) (S2^T zscale Q) / 2.  zscale = hd^-1/2 where the reference scales q before
 * the product (DETR), 1 where it divides the scores afterwards (LXMERT, VisualBERT). */
int mmx_lrp_attn_qk(const float* cam1, int ldA, const float* Q, int ldq, const float* K, int ldk, float zscale, float* cam_Q,
                    int ldcq, float* cam_K, int ldck, int B, int H, int T, int S, int hd, void* stream);
/* scores = zscale * Q K^T and mask[b,h,i,j] = key_bias[b,j] in the [B,H,T,ldA] layout: the two inputs of the Add that
 * VisualBERT's BertSelfAttention.relprop sends the relevance through (BERT_ours.py:352-395).  mask / key_bias may be NULL. */
int mmx_lrp_attn_scores(const float* Q, int ldq, const float* K, int ldk, const float* key_bias, float zscale, float* scores,
                        float* mask, int ldA, int B, int H, int T, int S, int hd, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * DETR's evaluation losses (DETR/engine.py:174 `criterion(outputs, targets)`): HungarianMatcher (DETR/models/matcher.py)
 * and SetCriterion (DETR/models/detr.py:103-275, DETR/models/segmentation.py:172-215), for the last decoder layer and the
 * auxiliary ones (DETR.forward's aux_outputs, detr.py:70-77, 95-100).  Shared layout: L layers (layer 0 the model's final
 * output, 1 .. L-1 aux_outputs 0 .. L-2; logits / boxes: host arrays of L device pointers to [B,Q,C1] and [B,Q,4]
 * contiguous fp32), B <= 64 images, Q queries.  The targets of all images are concatenated: tgt_ids [T] int64, tgt_boxes
 * [T,4] cxcywh fp32; tgt_offsets is a HOST array [B+1] (0, ..., T), image b owning targets off[b] .. off[b+1].
 * cost: the [Q, T_b] block of (layer l, image b) at l*Q*T + Q*off[b], row-major (the blocks kept after C.split(sizes),
 * matcher.py:80-81).  indices [L,2,T] int64: indices[l][0][off[b]+k] the query (ascending) and indices[l][1][off[b]+k]
 * the target of pair k < min(Q, T_b); unused slots -1.  Nothing here waits for the device.
 * ------------------------------------------------------------------------------------------------------- */
/* C = w_bbox cdist_L1 + w_class (-softmax(logits)[:, tgt_ids]) + w_giou (-GIoU) (matcher.py:60-77): the softmax in
 * mmx_detr_postprocess's order, GIoU in box_ops' order (DETR/util/box_ops.py:22-68).  status [L] int (device, zeroed
 * here): bit 1 when a predicted box of layer l - or, in status[0], a target box - fails generalized_box_iou's
 * `x1 >= x0 and y1 >= y0` assert (box_ops.py:51-52, NaN included); bit 2 in status[0] for a label outside [0, C1). */
int mmx_detr_match_cost(const float* const* logits, const float* const* boxes, int L, int B, int Q, int C1,
                        const int64_t* tgt_ids, const float* tgt_boxes, const int* tgt_offsets, float w_class, float w_bbox,
                        float w_giou, float* cost, int* status, void* stream);
/* scipy.optimize.linear_sum_assignment (matcher.py:81) of every (layer, image) cost block in one launch, one CTA each: the
 * shortest-augmenting-path algorithm scipy implements (Crouse 2016) restated in double, with its transpose of a tall
 * matrix, row order, column scan order, tie rule and dual updates, so ties resolve as scipy resolves them.  Q and every
 * T_b at most 1024.  status [L*B] int (device, zeroed here): 1 = a NaN or -inf entry ("matrix contains invalid numeric
 * entries"), 2 = no finite complete assignment ("cost matrix is infeasible"). */
int mmx_detr_match_lsa(const float* cost, int L, int B, int Q, const int* tgt_offsets, int64_t* indices, int* status,
                       void* stream);
/* The box and label losses of every layer (detr.py:124-188): out [L,5] = loss_ce (F.cross_entropy with empty_weight [C1]
 * over the B*Q rows, unmatched rows taking class C1-1), class_error (100 - top-1 accuracy of the matched rows, 100 when
 * none; util/misc.py:432-447; the top-1 is CUDA topk(1)'s: the lowest index among equal maxima, NaN above numbers), loss_bbox (sum |src - tgt| / num_boxes), loss_giou (sum (1 - GIoU) / num_boxes),
 * cardinality_error (mean over images of |#(argmax != C1-1) - T_b|).  num_boxes: one device float (detr.py:248-252).
 * Sums are doubles reduced in a fixed order. */
int mmx_detr_set_losses(const float* const* logits, const float* const* boxes, int L, int B, int Q, int C1,
                        const int64_t* tgt_ids, const float* tgt_boxes, const int* tgt_offsets, const int64_t* indices,
                        const float* empty_weight, const float* num_boxes, float* out, void* stream);
/* loss_masks (DETR/models/detr.py:184-211; focal and dice, segmentation.py:172-215) of one layer: each matched query's
 * pred_masks [B,Q,h,w] plane upsampled bilinearly (align_corners=False, ATen's arithmetic) to the padded target size
 * (max H_b, max W_b), the target read in place from tgt_masks[b] ([T_b, H_b, W_b], tgt_hw host [2B]; uint8 / bool for mask_dtype 0, fp32 for 1) and zero beyond its
 * image; out [2] = sigmoid focal loss (alpha 0.25, gamma 2, mean over pixels) and dice loss, each summed over the masks and
 * divided by num_boxes; both 0 when no image has a target.  indices: the [2,T] block of the layer.  Per-mask partial sums are doubles in a fixed order. */
int mmx_detr_mask_losses(const float* pred_masks, int B, int Q, int h, int w, const void* const* tgt_masks, const int* tgt_hw,
                         int mask_dtype, const int* tgt_offsets, const int64_t* indices, const float* num_boxes, float* out,
                         void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * Visualisation: the notebooks' last step, a relevance map turned into the picture a person looks at.  One launch per
 * call (one thread-block cluster per picture), no host synchronisation, no float atomics: deterministic and capturable.
 * ------------------------------------------------------------------------------------------------------- */
/* show_image_relevance (CLIP_explainability.ipynb:216) and generate_visualization (Transformer_MM_explainability_ViT.ipynb
 * :1223,1234): rel [B, h*w] fp32, images [n_img in {1, B}, 3, H, W] fp32 NCHW, out [B, H, W, 3] uint8.  Per map:
 * F.interpolate(bilinear, align_corners=False) to H x W with ATen's CUDA arithmetic (source scales scale_h / scale_w:
 * 1 / scale_factor, or (float)in / out for a size), a copy when the sizes are equal; min-max of the map and of the image
 * (all three channels); q = uint8(255 m) (truncation, NaN -> 0); cam = JET[q] / 255 + img, BGR channel c with RGB
 * channel c; vis = cam / max(cam) (NaN propagates); out = uint8(255 vis) with RGB <-> BGR swapped (cv2.cvtColor).
 * The JET table is cv2's COLORMAP_JET, held in the library.  h * w <= 4096 unless (h, w) = (H, W). */
int mmx_relevance_overlay(const float* rel, int B, int h, int w, float scale_h, float scale_w, const float* images, int n_img,
                          int H, int W, unsigned char* out, void* stream);
/* save_image_vis (LXMERT.ipynb:121, Transformer_MM_Explainability.ipynb:2571): img [n_img in {1, B}, H, W, 3] uint8 BGR,
 * boxes [B, n_boxes, 4] fp32 pixels (x0, y0, x1, y1), scores [B, n_boxes], out [B, H, W, 3] uint8 (what cv2.imwrite
 * encodes).  Box i covers mask[int(y0):int(y1), int(x0):int(x1)] with Python slice rules (truncation, one wrap of a
 * negative bound, clamping, start >= stop empty) and sets it to torch.max(score, mask) (NaN propagates); the mask is
 * min-max normalised in fp32 and multiplied into the image; the product goes to 8 bits as OpenCV's convertTo does (round
 * half to even, saturate, NaN -> 0).  n_boxes <= 1024. */
int mmx_box_relevance_image(const unsigned char* img, int n_img, int H, int W, const float* boxes, const float* scores, int B,
                            int n_boxes, unsigned char* out, void* stream);
/* show_heatmap_on_text's text_scores (CLIP_explainability.ipynb:254): R_text [B, ctx, ctx], tokens [B, ctx] int32.
 * eot = first argmax of tokens[b]; lens[b] = max(eot - 1, 0); scores[b, j] = R_text[b, eot, 1 + j] / s for j < lens[b]
 * (0 beyond), s the slice's sum in double rounded once to fp32.  scores [B, ctx] fp32, lens [B] int32, both device. */
int mmx_clip_text_scores(const float* R_text, const int* tokens, int B, int ctx, float* scores, int* lens, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MMX_H_ */
