// CLIP relevancy engine: interpret() for a batch of (image, text) pairs as one device-side pipeline.
//   forward (both towers on their own streams, A_l staged) -> logit head + analytic d(features) ->
//   dgrad-only backward (dA_l staged) -> rule 5 over all active layers in one launch -> rule 6 chain.
// Reference path replaced: CLIP_explainability.ipynb:151-208 driving CLIP/clip/model.py + CLIP/clip/auxilary.py.
#include "gemm.cuh"
#include <map>
#include <string>
#include <vector>
#include <cmath>
#include <cstring>
#include <cstdlib>
#include <nvtx3/nvToolsExt.h>   // header-only NVTX v3 (ranges for `ncu --nvtx --nvtx-include "vision/backward/"`, Nsight Systems)

namespace mmx {

// Host-side NVTX range around the launches of one pipeline stage (no cost when no tool is attached).
struct NvtxRange {
  explicit NvtxRange(const char* name) { nvtxRangePushA(name); }
  ~NvtxRange() { nvtxRangePop(); }
  NvtxRange(const NvtxRange&) = delete;
  NvtxRange& operator=(const NvtxRange&) = delete;
};

// kernels from the other translation units
int layernorm_fwd(const float*, int, const int*, const float*, const float*, float*, int, float*, float*, int, int, float, cudaStream_t,
                  const int* rows_dev);
int layernorm_bwd(const float*, int, const float*, int, const int*, const float*, const float*, const float*, const float*, int,
                  float*, int, int, int, cudaStream_t, const int* rows_dev);
int attention_fwd(const float*, int, const float*, int, const float*, int, const float*, float*, int, float*, int, int, int, int,
                  int, int, float, int, cudaStream_t, const int* offs, const int* lens);
int attention_bwd(const float*, int, const float*, int, const float*, int, const float*, int, const float*, float*, int, float*,
                  float*, int, float*, int, float*, int, int, int, int, int, int, float, int, cudaStream_t, const int* offs,
                  const int* lens, const float* gscale);
int text_embed_packed(const int*, const float*, const float*, float*, int*, int*, int*, int*, int, int, int, int, cudaStream_t);
int avg_heads(const float*, const float*, float*, int, int, int, int, int, int, cudaStream_t);
int bmm_add(const float*, int, long long, int, const float*, int, long long, const float*, int, long long, float*, int, long long,
            int, int, int, int, int, cudaStream_t);
int self_update_tc(const float* Abar, int ld_a, const float* R, float* R_out, int ld, int B, int S, int Q, cudaStream_t st,
                   bool* taken);
bool rule6_chain_ok(int S, int ld, int ld_out, const float* Abar, const float* R_out);
int rule6_chain(const float* Abar, long long layer_stride, int ld, float* R_out, int ld_out, int B, int S, int L, cudaStream_t st);
int im2col_patches(const float*, float*, int, int, int, cudaStream_t);
int vision_tokens_lnpre(const float*, int, const float*, const float*, const float*, const float*, float*, int, int, int, float,
                        cudaStream_t);
int text_embed(const int*, const float*, const float*, float*, int*, int, int, int, int, cudaStream_t);
int cls_rows(int*, int, int, cudaStream_t);
int clip_head(const float*, const float*, float, float*, float*, float*, float*, float*, float*, float*, int, int, cudaStream_t);
int scale_inplace(float*, long long, float, cudaStream_t);
int set_eye(float*, int, int, int, cudaStream_t);
int slice_out(const float*, long long, int, int, int, float*, int, int, int, cudaStream_t);

__global__ void __launch_bounds__(256) transpose_kernel(const float* __restrict__ in, float* __restrict__ out, int rows, int cols) {
  __shared__ float t[32][33];
  const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int r = r0 + i, c = c0 + threadIdx.x;
    if (r < rows && c < cols) t[i][threadIdx.x] = in[(long long)r * cols + c];
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int c = c0 + i, r = r0 + threadIdx.x;
    if (r < rows && c < cols) out[(long long)c * rows + r] = t[threadIdx.x][i];
  }
}
static int transpose(const float* in, float* out, int rows, int cols, cudaStream_t st) {
  dim3 grid(cdiv(cols, 32), cdiv(rows, 32)), block(32, 8);
  transpose_kernel<<<grid, block, 0, st>>>(in, out, rows, cols);
  MMX_LAUNCH_CHECK();
  return 0;
}

// a K-major GEMM "B" operand [N,K]
struct Mat {
  float* w = nullptr;
  int N = 0, K = 0;
  void* packed = nullptr;   // fp16 hi / lo planes for the fp16x3 backend (built by finalize)
};

struct LayerW {
  float *ln1_g, *ln1_b, *ln2_g, *ln2_b;
  float *bqkv, *bo, *bfc, *bproj;
  Mat Wqkv, Wo, Wfc, Wproj;             // forward operands [out, in]
  Mat WqkvT, WoT, WfcT, WprojT;         // dgrad operands (W^T, K-major for the NT GEMM)
};

static inline int mm(const float* A, int lda, const Mat& B, float* C, int ldc, int M, const GemmEpilogue& ep, cudaStream_t st) {
  return gemm_nt_b(A, lda, packed_operand(B.w, B.K, B.packed, B.N, B.K), C, ldc, M, B.N, B.K, ep, st);
}

struct Tower {
  int L = 0, D = 0, H = 0, S = 0, ld = 0, hd = 0, act = MMX_ACT_QUICKGELU, causal = 0;
  std::vector<LayerW> w;
  // activation arena (sized for max batch Bm)
  float* x = nullptr;       // [L+1][M,D] residual stream (x[l] = input of block l)
  float* xmid = nullptr;    // [L][M,D]
  float* qkv = nullptr;     // [L][M,3D]
  float* f = nullptr;       // [L][M,4D]  MLP pre-activations
  float* stats = nullptr;   // [L][4][M]  mean1, rstd1, mean2, rstd2
  float* A = nullptr;       // [L][B,H,S,ld]   (layer stride uses the CURRENT batch)
  float* dA = nullptr;      // [L][B,H,S,ld]
  float* Abar = nullptr;    // [L][B,S,ld]
  float* R[2] = {nullptr, nullptr};  // [B,S,ld] ping-pong
  float *h = nullptr, *o = nullptr, *g = nullptr, *dx0 = nullptr, *dx1 = nullptr, *dqkv = nullptr, *delta = nullptr;
  int* rows = nullptr;      // [Bm] pooled row per sample (cls / eot)
  // ragged text batches: packed rows, sample b owns rows offs[b] .. offs[b] + lens[b] - 1; *total = sum(lens)
  bool ragged = false;
  int *offs = nullptr, *lens = nullptr, *total = nullptr;
  int rows_host = -1;       // sum(lens) read back for this chunk (-1: unknown, the GEMMs read *total on the device)
  float *pool_ln = nullptr, *pool_mean = nullptr, *pool_rstd = nullptr, *dpool = nullptr;  // [Bm,D], [Bm]
  float *lnf_g = nullptr, *lnf_b = nullptr;  // ln_post / ln_final
  Mat proj, projT;                           // [D,E] (as stored: the dgrad operand), [E,D] (forward operand)
  float *feat = nullptr, *featn = nullptr, *dfeat = nullptr;  // [Bm,E]
  float* gscale = nullptr;  // [Bm] power-of-two factor carried by this tower's gradient stream (per sample)
  cudaStream_t st = nullptr;
  long long M(int B) const { return (long long)B * S; }
};

}  // namespace mmx

using namespace mmx;

struct mmx_clip {
  mmx_clip_config cfg;
  int Bm = 0;
  int G = 0, E = 0;
  Tower v, t;
  float logit_scale = 0.f;
  // named tensors
  struct Slot { float* ptr; size_t numel; bool loaded; };
  std::map<std::string, Slot> slots;
  std::vector<void*> allocs;
  bool finalized = false;
  // vision pre
  Mat conv_w;
  float *cls = nullptr, *pos_v = nullptr, *lnpre_g = nullptr, *lnpre_b = nullptr;
  float *patches = nullptr, *patch_emb = nullptr;
  // text pre
  float *tok_emb = nullptr, *pos_t = nullptr;
  // io staging (host entry point)
  float* d_images = nullptr; int32_t* d_tokens = nullptr; float *d_Rtext = nullptr, *d_Rimage = nullptr;
  float *logits = nullptr, *diag = nullptr;
  cudaStream_t main = nullptr;
  cudaEvent_t ev_fork = nullptr, ev_v = nullptr, ev_t = nullptr, ev_head = nullptr, ev_rows = nullptr;
  int* rows_pinned = nullptr;   // host copy of the text tower's packed row count (ragged batches)
  cudaStream_t text_stream = nullptr;   // the text tower's own stream (h->t.st aliases the vision stream in serial mode)
  int lastB = 0, last_start_v = 0, last_start_t = 0;
  size_t bytes = 0;
};

namespace {

int dalloc(mmx_clip* h, void** p, size_t bytes) {
  MMX_CHECK_CUDA(cudaMalloc(p, bytes ? bytes : 16));
  h->allocs.push_back(*p);
  h->bytes += bytes;
  return 0;
}
template <typename T>
int dallocT(mmx_clip* h, T** p, size_t n) { return dalloc(h, (void**)p, n * sizeof(T)); }

int reg(mmx_clip* h, const std::string& name, float** p, size_t numel) {
  MMX_TRY(dallocT(h, p, numel));
  h->slots[name] = {*p, numel, false};
  return 0;
}

int alloc_tower(mmx_clip* h, Tower& T, const std::string& prefix, int Bm, int E) {
  const size_t M = (size_t)Bm * T.S, D = T.D, L = T.L;
  T.ld = round_up(T.S, 4);
  T.hd = T.D / T.H;
  T.w.resize(L);
  for (size_t l = 0; l < L; ++l) {
    LayerW& w = T.w[l];
    const std::string p = prefix + "resblocks." + std::to_string(l) + ".";
    MMX_TRY(reg(h, p + "ln_1.weight", &w.ln1_g, D));
    MMX_TRY(reg(h, p + "ln_1.bias", &w.ln1_b, D));
    MMX_TRY(reg(h, p + "ln_2.weight", &w.ln2_g, D));
    MMX_TRY(reg(h, p + "ln_2.bias", &w.ln2_b, D));
    MMX_TRY(reg(h, p + "attn.in_proj_weight", &w.Wqkv.w, 3 * D * D));
    MMX_TRY(reg(h, p + "attn.in_proj_bias", &w.bqkv, 3 * D));
    MMX_TRY(reg(h, p + "attn.out_proj.weight", &w.Wo.w, D * D));
    MMX_TRY(reg(h, p + "attn.out_proj.bias", &w.bo, D));
    MMX_TRY(reg(h, p + "mlp.c_fc.weight", &w.Wfc.w, 4 * D * D));
    MMX_TRY(reg(h, p + "mlp.c_fc.bias", &w.bfc, 4 * D));
    MMX_TRY(reg(h, p + "mlp.c_proj.weight", &w.Wproj.w, 4 * D * D));
    MMX_TRY(reg(h, p + "mlp.c_proj.bias", &w.bproj, D));
    MMX_TRY(dallocT(h, &w.WqkvT.w, 3 * D * D));
    MMX_TRY(dallocT(h, &w.WoT.w, D * D));
    MMX_TRY(dallocT(h, &w.WfcT.w, 4 * D * D));
    MMX_TRY(dallocT(h, &w.WprojT.w, 4 * D * D));
    const int Di = (int)D;
    w.Wqkv.N = 3 * Di; w.Wqkv.K = Di; w.WqkvT.N = Di; w.WqkvT.K = 3 * Di;
    w.Wo.N = Di; w.Wo.K = Di; w.WoT.N = Di; w.WoT.K = Di;
    w.Wfc.N = 4 * Di; w.Wfc.K = Di; w.WfcT.N = Di; w.WfcT.K = 4 * Di;
    w.Wproj.N = Di; w.Wproj.K = 4 * Di; w.WprojT.N = 4 * Di; w.WprojT.K = Di;
  }
  MMX_TRY(dallocT(h, &T.x, (L + 1) * M * D));
  MMX_TRY(dallocT(h, &T.xmid, L * M * D));
  MMX_TRY(dallocT(h, &T.qkv, L * M * 3 * D));
  MMX_TRY(dallocT(h, &T.f, L * M * 4 * D));
  MMX_TRY(dallocT(h, &T.stats, L * 4 * M));
  const size_t plane = (size_t)Bm * T.H * T.S * T.ld;
  MMX_TRY(dallocT(h, &T.A, L * plane));
  MMX_TRY(dallocT(h, &T.dA, L * plane));
  MMX_TRY(dallocT(h, &T.Abar, L * (size_t)Bm * T.S * T.ld));
  MMX_TRY(dallocT(h, &T.R[0], (size_t)Bm * T.S * T.ld));
  MMX_TRY(dallocT(h, &T.R[1], (size_t)Bm * T.S * T.ld));
  MMX_TRY(dallocT(h, &T.h, M * D));
  MMX_TRY(dallocT(h, &T.o, M * D));
  MMX_TRY(dallocT(h, &T.g, M * 4 * D));
  MMX_TRY(dallocT(h, &T.dx0, M * D));
  MMX_TRY(dallocT(h, &T.dx1, M * D));
  MMX_TRY(dallocT(h, &T.dqkv, M * 3 * D));
  MMX_TRY(dallocT(h, &T.delta, (size_t)Bm * T.H * T.S));
  MMX_TRY(dallocT(h, &T.rows, (size_t)Bm));
  MMX_TRY(dallocT(h, &T.offs, (size_t)Bm));
  MMX_TRY(dallocT(h, &T.lens, (size_t)Bm));
  MMX_TRY(dallocT(h, &T.total, (size_t)1));
  MMX_TRY(dallocT(h, &T.pool_ln, (size_t)Bm * D));
  MMX_TRY(dallocT(h, &T.pool_mean, (size_t)Bm));
  MMX_TRY(dallocT(h, &T.pool_rstd, (size_t)Bm));
  MMX_TRY(dallocT(h, &T.dpool, (size_t)Bm * D));
  MMX_TRY(dallocT(h, &T.projT.w, (size_t)E * D));
  T.proj.N = (int)D; T.proj.K = E; T.projT.N = E; T.projT.K = (int)D;
  MMX_TRY(dallocT(h, &T.feat, (size_t)Bm * E));
  MMX_TRY(dallocT(h, &T.featn, (size_t)Bm * E));
  MMX_TRY(dallocT(h, &T.dfeat, (size_t)Bm * E));
  MMX_TRY(dallocT(h, &T.gscale, (size_t)Bm));
  MMX_CHECK_CUDA(cudaStreamCreateWithFlags(&T.st, cudaStreamNonBlocking));
  return 0;
}

// ---- tower forward / backward ---------------------------------------------------------------------------
int tower_forward(Tower& T, int B) {
  cudaStream_t st = T.st;
  const int M = (int)T.M(B), D = T.D;
  const size_t MD = (size_t)M * D;
  const size_t plane = (size_t)B * T.H * T.S * T.ld;
  const float scale = 1.f / sqrtf((float)T.hd);     // CLIP/clip/auxilary.py:72
  const int* md = T.ragged ? T.total : nullptr;      // device row count; M = B*S is then only the upper bound
  const int* offs = T.ragged ? T.offs : nullptr;
  const int* lens = T.ragged ? T.lens : nullptr;
  // GEMM row count: exact on the host when the packed row count was read back (tile width / grid chosen for the real
  // size), else the upper bound with the device-side count
  const int Mg = (T.ragged && T.rows_host >= 0) ? T.rows_host : M;
  const int* mg = (T.ragged && T.rows_host >= 0) ? nullptr : md;
  for (int l = 0; l < T.L; ++l) {
    const LayerW& w = T.w[l];
    float* x_in = T.x + l * MD;
    float* x_mid = T.xmid + l * MD;
    float* x_out = T.x + (l + 1) * MD;
    float* qkv = T.qkv + l * MD * 3;
    float* f = T.f + l * MD * 4;
    float* stt = T.stats + (size_t)l * 4 * M;
    MMX_TRY(layernorm_fwd(x_in, D, nullptr, w.ln1_g, w.ln1_b, T.h, D, stt, stt + M, M, D, 1e-5f, st, md));
    GemmEpilogue e1; e1.bias = w.bqkv; e1.m_dev = mg;
    MMX_TRY(mm(T.h, D, w.Wqkv, qkv, 3 * D, Mg, e1, st));
    MMX_TRY(attention_fwd(qkv, 3 * D, qkv + D, 3 * D, qkv + 2 * D, 3 * D, nullptr, T.A + l * plane, T.ld, T.o, D, B, T.H, T.S,
                          T.S, T.hd, scale, T.causal ? MMX_ATTN_CAUSAL : 0, st, offs, lens));
    GemmEpilogue e2; e2.bias = w.bo; e2.residual = x_in; e2.ldres = D; e2.m_dev = mg;
    MMX_TRY(mm(T.o, D, w.Wo, x_mid, D, Mg, e2, st));
    MMX_TRY(layernorm_fwd(x_mid, D, nullptr, w.ln2_g, w.ln2_b, T.h, D, stt + 2 * M, stt + 3 * M, M, D, 1e-5f, st, md));
    // fc2 takes act(f).  Where its split pass can apply the activation (backend 3), act(f) never goes through HBM: fc1
    // stores f only.  Elsewhere fc1's epilogue also stores g = act(f), and fc2 reads g.  Same bits either way.
    GemmEpilogue e4; e4.bias = w.bproj; e4.residual = x_mid; e4.ldres = D; e4.m_dev = mg; e4.a_act = T.act;
    const bool act_in_split = gemm_a_act_ok(f, 4 * D, packed_operand(w.Wproj.w, w.Wproj.K, w.Wproj.packed, w.Wproj.N, w.Wproj.K),
                                            x_out, D, w.Wproj.N, w.Wproj.K, e4);
    if (!act_in_split) e4.a_act = MMX_ACT_NONE;
    GemmEpilogue e3; e3.bias = w.bfc; e3.C_act = act_in_split ? nullptr : T.g; e3.act = T.act; e3.m_dev = mg;
    MMX_TRY(mm(T.h, D, w.Wfc, f, 4 * D, Mg, e3, st));
    MMX_TRY(mm(act_in_split ? f : T.g, 4 * D, w.Wproj, x_out, D, Mg, e4, st));
  }
  return 0;
}

// pooled feature: feat = LN(x_L[rows]) @ proj
int tower_pool(Tower& T, int B, int E) {
  const size_t MD = (size_t)T.M(B) * T.D;
  const float* xL = T.x + (size_t)T.L * MD;
  MMX_TRY(layernorm_fwd(xL, T.D, T.rows, T.lnf_g, T.lnf_b, T.pool_ln, T.D, T.pool_mean, T.pool_rstd, B, T.D, 1e-5f, T.st, nullptr));
  GemmEpilogue e;
  MMX_TRY(mm(T.pool_ln, T.D, T.projT, T.feat, E, B, e, T.st));
  return 0;
}

// backward from dfeat down to block `stop` (its dA is the last thing computed)
int tower_backward(Tower& T, int B, int E, int stop) {
  cudaStream_t st = T.st;
  const int M = (int)T.M(B), D = T.D;
  const size_t MD = (size_t)M * D;
  const size_t plane = (size_t)B * T.H * T.S * T.ld;
  const float scale = 1.f / sqrtf((float)T.hd);
  GemmEpilogue e0;
  MMX_TRY(mm(T.dfeat, E, T.proj, T.dpool, D, B, e0, st));                          // d(LN out) = dfeat @ proj^T
  float* dx_out = T.dx0;
  float* dx_mid = T.dx1;
  MMX_CHECK_CUDA(cudaMemsetAsync(dx_out, 0, MD * sizeof(float), st));
  MMX_TRY(layernorm_bwd(T.dpool, D, T.x + (size_t)T.L * MD, D, T.rows, T.lnf_g, T.pool_mean, T.pool_rstd, nullptr, 0, dx_out, D,
                        B, D, st, nullptr));
  const int* md = T.ragged ? T.total : nullptr;
  const int* offs = T.ragged ? T.offs : nullptr;
  const int* lens = T.ragged ? T.lens : nullptr;
  const int Mg = (T.ragged && T.rows_host >= 0) ? T.rows_host : M;
  const int* mg = (T.ragged && T.rows_host >= 0) ? nullptr : md;
  for (int l = T.L - 1; l >= stop; --l) {
    const LayerW& w = T.w[l];
    const float* x_in = T.x + l * MD;
    const float* x_mid = T.xmid + l * MD;
    const float* qkv = T.qkv + l * MD * 3;
    const float* f = T.f + l * MD * 4;
    const float* stt = T.stats + (size_t)l * 4 * M;
    GemmEpilogue e1; e1.pre = f; e1.ldpre = 4 * D; e1.act = T.act; e1.m_dev = mg;
    MMX_TRY(mm(dx_out, D, w.WprojT, T.g, 4 * D, Mg, e1, st));                        // df = (dx W_proj) . act'(f)
    GemmEpilogue e2; e2.m_dev = mg;
    MMX_TRY(mm(T.g, 4 * D, w.WfcT, T.h, D, Mg, e2, st));                             // dh2 = df W_fc
    MMX_TRY(layernorm_bwd(T.h, D, x_mid, D, nullptr, w.ln2_g, stt + 2 * M, stt + 3 * M, dx_out, D, dx_mid, D, M, D, st, md));
    MMX_TRY(mm(dx_mid, D, w.WoT, T.o, D, Mg, e2, st));                               // d(attn out) = dx_mid W_o
    const bool last = (l == stop);
    MMX_TRY(attention_bwd(T.o, D, qkv, 3 * D, qkv + D, 3 * D, qkv + 2 * D, 3 * D, T.A + l * plane, T.dA + l * plane, T.ld,
                          T.delta, last ? nullptr : T.dqkv, 3 * D, last ? nullptr : T.dqkv + D, 3 * D,
                          last ? nullptr : T.dqkv + 2 * D, 3 * D, B, T.H, T.S, T.S, T.hd, scale, 0, st, offs, lens, T.gscale));
    if (last) break;
    MMX_TRY(mm(T.dqkv, 3 * D, w.WqkvT, T.h, D, Mg, e2, st));                          // dh1 = dqkv W_qkv
    MMX_TRY(layernorm_bwd(T.h, D, x_in, D, nullptr, w.ln1_g, stt, stt + M, dx_mid, D, dx_out, D, M, D, st, md));
  }
  return 0;
}

// rule 5 over layers [start, L) in one launch, then the rule-6 chain.  Returns the index of the R buffer.
int tower_rules(Tower& T, int B, int start, int* r_idx) {
  cudaStream_t st = T.st;
  const size_t plane = (size_t)B * T.H * T.S * T.ld;
  const size_t bplane = (size_t)B * T.S * T.ld;
  const int nl = T.L - start;
  // padded rows (ld) are zero in A and dA, so the plane is treated as dense [S, ld]
  MMX_TRY(avg_heads(T.A + start * plane, T.dA + start * plane, T.Abar + start * bplane, nl * B, T.H, T.S, T.ld, T.ld, T.ld, st));
  if (rule6_chain_ok(T.S, T.ld, T.ld, T.Abar + start * bplane, T.R[0])) {
    // the whole chain R = I; R <- R + Abar_l R in one launch, R resident in shared memory (rule_chain.cu)
    MMX_TRY(rule6_chain(T.Abar + start * bplane, (long long)bplane, T.ld, T.R[0], T.ld, B, T.S, nl, st));
    *r_idx = 0;
    return 0;
  }
  MMX_TRY(set_eye(T.R[0], B, T.S, T.ld, st));
  int cur = 0;
  const long long sp = (long long)T.S * T.ld;
  for (int l = start; l < T.L; ++l) {
    bool tc = false;   // S >= 128 (ViT-B/16 197, L/14 257, L/14@336 577): the batched wgmma rule GEMM
    MMX_TRY(self_update_tc(T.Abar + l * bplane, T.ld, T.R[cur], T.R[cur ^ 1], T.ld, B, T.S, T.S, st, &tc));
    if (!tc)
      MMX_TRY(bmm_add(T.Abar + l * bplane, T.ld, sp, 0, T.R[cur], T.ld, sp, T.R[cur], T.ld, sp, T.R[cur ^ 1], T.ld, sp, B, T.S,
                      T.ld, T.S, 0, st));
    cur ^= 1;
  }
  *r_idx = cur;
  return 0;
}

int run_chunk(mmx_clip* h, const float* images, int n_images, const int32_t* tokens, int B, int start_v, int start_t,
              float* R_text, float* R_image, cudaStream_t caller) {
  const mmx_clip_config& c = h->cfg;
  Tower &V = h->v, &Tx = h->t;
  const int E = h->E;
  MMX_CHECK_CUDA(cudaEventRecord(h->ev_fork, caller));
  MMX_CHECK_CUDA(cudaStreamWaitEvent(V.st, h->ev_fork, 0));
  MMX_CHECK_CUDA(cudaStreamWaitEvent(Tx.st, h->ev_fork, 0));
  // ---- text embedding first: it yields the packed row count of the ragged text batch, which is copied to the host
  // while the vision tower's launches are being enqueued (no stall), so the text GEMMs get exact sizes
  if (Tx.ragged) {
    MMX_TRY(text_embed_packed(tokens, h->tok_emb, h->pos_t, Tx.x, Tx.offs, Tx.lens, Tx.rows, Tx.total, B, Tx.S, Tx.D,
                              c.vocab_size, Tx.st));
    MMX_CHECK_CUDA(cudaMemcpyAsync(h->rows_pinned, Tx.total, sizeof(int), cudaMemcpyDeviceToHost, Tx.st));
    MMX_CHECK_CUDA(cudaEventRecord(h->ev_rows, Tx.st));
  } else {
    MMX_TRY(text_embed(tokens, h->tok_emb, h->pos_t, Tx.x, Tx.rows, B, Tx.S, Tx.D, c.vocab_size, Tx.st));
  }
  // ---- vision tower
  {
    NvtxRange r("vision/forward");
    const int p = c.vision_patch_size, G = h->G, Kp = 3 * p * p;
    MMX_TRY(im2col_patches(images, h->patches, n_images, c.image_resolution, p, V.st));
    GemmEpilogue e;
    MMX_TRY(mm(h->patches, Kp, h->conv_w, h->patch_emb, V.D, n_images * G * G, e, V.st));
    MMX_TRY(vision_tokens_lnpre(h->patch_emb, n_images, h->cls, h->pos_v, h->lnpre_g, h->lnpre_b, V.x, B, V.S, V.D, 1e-5f, V.st));
    MMX_TRY(cls_rows(V.rows, B, V.S, V.st));
    MMX_TRY(tower_forward(V, B));
    MMX_TRY(tower_pool(V, B, E));
  }
  // ---- text tower
  {
    NvtxRange r("text/forward");
    Tx.rows_host = -1;
    if (Tx.ragged) {
      MMX_CHECK_CUDA(cudaEventSynchronize(h->ev_rows));
      Tx.rows_host = *h->rows_pinned;
      MMX_REQUIRE(Tx.rows_host >= 0 && Tx.rows_host <= B * Tx.S, "packed text row count out of range");
    }
    MMX_TRY(tower_forward(Tx, B));
    MMX_TRY(tower_pool(Tx, B, E));
  }
  // ---- head on the vision stream after the text features landed
  MMX_CHECK_CUDA(cudaEventRecord(h->ev_t, Tx.st));
  MMX_CHECK_CUDA(cudaStreamWaitEvent(V.st, h->ev_t, 0));
  MMX_TRY(clip_head(V.feat, Tx.feat, expf(h->logit_scale), V.featn, Tx.featn, V.dfeat, Tx.dfeat, h->diag, V.gscale, Tx.gscale, B,
                    E, V.st));
  MMX_CHECK_CUDA(cudaEventRecord(h->ev_head, V.st));
  MMX_CHECK_CUDA(cudaStreamWaitEvent(Tx.st, h->ev_head, 0));
  {
    GemmEpilogue e;   // logits_per_image [B,B] (CLIP/clip/model.py:373); not needed by the rule, kept for API parity/tests
    MMX_TRY(gemm_nt(V.featn, E, Tx.featn, E, h->logits, B, B, B, E, e, V.st));
    MMX_TRY(scale_inplace(h->logits, (long long)B * B, expf(h->logit_scale), V.st));
  }
  // ---- backward + rules, towers independent again
  int rv = 0, rt = 0;
  {
    NvtxRange r("vision/backward");
    MMX_TRY(tower_backward(V, B, E, start_v));
  }
  {
    NvtxRange r("vision/rules");
    MMX_TRY(tower_rules(V, B, start_v, &rv));
    MMX_TRY(slice_out(V.R[rv], (long long)V.S * V.ld, V.ld, 0, 1, R_image, B, 1, V.S - 1, V.st));       // R[:,0,1:]
  }
  {
    NvtxRange r("text/backward");
    MMX_TRY(tower_backward(Tx, B, E, start_t));
  }
  {
    NvtxRange r("text/rules");
    MMX_TRY(tower_rules(Tx, B, start_t, &rt));
    MMX_TRY(slice_out(Tx.R[rt], (long long)Tx.S * Tx.ld, Tx.ld, 0, 0, R_text, B, Tx.S, Tx.S, Tx.st));
  }
  MMX_CHECK_CUDA(cudaEventRecord(h->ev_v, V.st));
  MMX_CHECK_CUDA(cudaEventRecord(h->ev_t, Tx.st));
  MMX_CHECK_CUDA(cudaStreamWaitEvent(caller, h->ev_v, 0));
  MMX_CHECK_CUDA(cudaStreamWaitEvent(caller, h->ev_t, 0));
  return 0;
}

int resolve_start(int start, int L, int* out) {
  if (start == -1) start = L - 1;                                   // CLIP_explainability.ipynb:165-167
  MMX_REQUIRE(start >= 0 && start < L, "start_layer out of range");
  *out = start;
  return 0;
}

}  // namespace

extern "C" {

int mmx_clip_create(const mmx_clip_config* cfg, int max_batch, mmx_clip** out) {
  MMX_REQUIRE(cfg && out && max_batch > 0, "bad arguments");
  int ndev = 0;
  MMX_CHECK_CUDA(cudaGetDeviceCount(&ndev));
  MMX_REQUIRE(ndev > 0, "no CUDA device");
  MMX_REQUIRE(cfg->vision_width % 64 == 0, "vision width must be a multiple of 64 (heads = width/64)");
  MMX_REQUIRE(cfg->transformer_width % cfg->transformer_heads == 0, "text width % heads");
  MMX_REQUIRE(cfg->image_resolution % cfg->vision_patch_size == 0, "resolution % patch");
  MMX_REQUIRE(cfg->vision_width % 4 == 0 && cfg->transformer_width % 4 == 0 && cfg->embed_dim % 4 == 0, "dims % 4");
  mmx_clip* h = new mmx_clip();
  h->cfg = *cfg;
  h->Bm = max_batch;
  h->G = cfg->image_resolution / cfg->vision_patch_size;
  h->E = cfg->embed_dim;
  Tower &V = h->v, &T = h->t;
  V.L = cfg->vision_layers; V.D = cfg->vision_width; V.H = cfg->vision_width / 64; V.S = h->G * h->G + 1; V.causal = 0;
  T.L = cfg->transformer_layers; T.D = cfg->transformer_width; T.H = cfg->transformer_heads; T.S = cfg->context_length;
  T.causal = 1;
  {
    // tokens after the EOT are dead under the causal mask (see norm_embed.cu: text_lens_kernel); MMX_RAGGED_TEXT=0
    // restores the reference's dense [B,77] computation (same results)
    const char* e = getenv("MMX_RAGGED_TEXT");
    T.ragged = !(e && atoi(e) == 0);
  }
  const int hdv = V.D / V.H, hdt = T.D / T.H;
  int rc = 0;
  auto fail = [&](int r) { mmx_clip_destroy(h); return r; };
  if (!((hdv == 16 || hdv == 32 || hdv == 64) && (hdt == 16 || hdt == 32 || hdt == 64))) {
    set_error("head_dim must be 16, 32 or 64");
    return fail(2);
  }
  const int Kp = 3 * cfg->vision_patch_size * cfg->vision_patch_size;
  if ((rc = alloc_tower(h, V, "visual.transformer.", max_batch, h->E))) return fail(rc);
  if ((rc = alloc_tower(h, T, "transformer.", max_batch, h->E))) return fail(rc);
#define REG(name, ptr, n) if ((rc = reg(h, name, ptr, n))) return fail(rc)
#define ALLOC(ptr, n) if ((rc = dallocT(h, ptr, n))) return fail(rc)
  REG("visual.conv1.weight", &h->conv_w.w, (size_t)V.D * Kp);
  h->conv_w.N = V.D; h->conv_w.K = Kp;
  REG("visual.class_embedding", &h->cls, V.D);
  REG("visual.positional_embedding", &h->pos_v, (size_t)V.S * V.D);
  REG("visual.ln_pre.weight", &h->lnpre_g, V.D);
  REG("visual.ln_pre.bias", &h->lnpre_b, V.D);
  REG("visual.ln_post.weight", &V.lnf_g, V.D);
  REG("visual.ln_post.bias", &V.lnf_b, V.D);
  REG("visual.proj", &V.proj.w, (size_t)V.D * h->E);
  REG("token_embedding.weight", &h->tok_emb, (size_t)cfg->vocab_size * T.D);
  REG("positional_embedding", &h->pos_t, (size_t)T.S * T.D);
  REG("ln_final.weight", &T.lnf_g, T.D);
  REG("ln_final.bias", &T.lnf_b, T.D);
  REG("text_projection", &T.proj.w, (size_t)T.D * h->E);
  ALLOC(&h->patches, (size_t)max_batch * h->G * h->G * Kp);
  ALLOC(&h->patch_emb, (size_t)max_batch * h->G * h->G * V.D);
  ALLOC(&h->logits, (size_t)max_batch * max_batch);
  ALLOC(&h->diag, (size_t)max_batch);
  ALLOC(&h->d_images, (size_t)max_batch * 3 * cfg->image_resolution * cfg->image_resolution);
  ALLOC(&h->d_tokens, (size_t)max_batch * T.S);
  ALLOC(&h->d_Rtext, (size_t)max_batch * T.S * T.S);
  ALLOC(&h->d_Rimage, (size_t)max_batch * (V.S - 1));
#undef REG
#undef ALLOC
  h->slots["logit_scale"] = {nullptr, 1, false};
  if (cudaStreamCreateWithFlags(&h->main, cudaStreamNonBlocking) != cudaSuccess ||
      cudaEventCreateWithFlags(&h->ev_fork, cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreateWithFlags(&h->ev_v, cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreateWithFlags(&h->ev_t, cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreateWithFlags(&h->ev_head, cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreateWithFlags(&h->ev_rows, cudaEventDisableTiming) != cudaSuccess ||
      cudaHostAlloc((void**)&h->rows_pinned, sizeof(int), cudaHostAllocDefault) != cudaSuccess) {
    set_error("stream/event creation failed");
    return fail(1);
  }
  h->text_stream = h->t.st;
  *out = h;
  return 0;
}

int mmx_clip_set_serial(mmx_clip* h, int serial) {
  MMX_REQUIRE(h, "null handle");
  MMX_CHECK_CUDA(cudaDeviceSynchronize());
  h->t.st = serial ? h->v.st : h->text_stream;
  return 0;
}

void mmx_clip_destroy(mmx_clip* h) {
  if (!h) return;
  cudaDeviceSynchronize();
  for (void* p : h->allocs) cudaFree(p);
  h->t.st = h->text_stream;
  if (h->v.st) cudaStreamDestroy(h->v.st);
  if (h->t.st) cudaStreamDestroy(h->t.st);
  if (h->main) cudaStreamDestroy(h->main);
  for (cudaEvent_t e : {h->ev_fork, h->ev_v, h->ev_t, h->ev_head, h->ev_rows}) if (e) cudaEventDestroy(e);
  if (h->rows_pinned) cudaFreeHost(h->rows_pinned);
  delete h;
}

int mmx_clip_load_tensor(mmx_clip* h, const char* name, const float* data, size_t numel) {
  MMX_REQUIRE(h && name && data, "bad arguments");
  auto it = h->slots.find(name);
  MMX_REQUIRE(it != h->slots.end(), std::string("unknown tensor name: ") + name);
  MMX_REQUIRE(it->second.numel == numel, std::string("size mismatch for ") + name + ": expected " +
                                             std::to_string(it->second.numel) + ", got " + std::to_string(numel));
  if (it->first == "logit_scale") {
    h->logit_scale = data[0];
  } else {
    MMX_CHECK_CUDA(cudaMemcpy(it->second.ptr, data, numel * sizeof(float), cudaMemcpyHostToDevice));
  }
  it->second.loaded = true;
  h->finalized = false;
  return 0;
}

int mmx_clip_finalize(mmx_clip* h) {
  MMX_REQUIRE(h, "null handle");
  for (auto& kv : h->slots) MMX_REQUIRE(kv.second.loaded, std::string("tensor not loaded: ") + kv.first);
  cudaStream_t st = h->main;
  for (Tower* T : {&h->v, &h->t}) {
    const int D = T->D;
    for (LayerW& w : T->w) {
      MMX_TRY(transpose(w.Wqkv.w, w.WqkvT.w, 3 * D, D, st));    // [3D,D] -> [D,3D]
      MMX_TRY(transpose(w.Wo.w, w.WoT.w, D, D, st));
      MMX_TRY(transpose(w.Wfc.w, w.WfcT.w, 4 * D, D, st));      // [4D,D] -> [D,4D]
      MMX_TRY(transpose(w.Wproj.w, w.WprojT.w, D, 4 * D, st));  // [D,4D] -> [4D,D]
    }
    MMX_TRY(transpose(T->proj.w, T->projT.w, D, h->E, st));     // [D,E] -> [E,D]
  }
  // fp16 hi / lo planes of every static GEMM operand (the fp16x3 backend; 4 bytes per element like the fp32 copy)
  if (gemm_tc_available()) {
    std::vector<Mat*> mats{&h->conv_w};
    for (Tower* T : {&h->v, &h->t}) {
      for (LayerW& w : T->w)
        for (Mat* m : {&w.Wqkv, &w.Wo, &w.Wfc, &w.Wproj, &w.WqkvT, &w.WoT, &w.WfcT, &w.WprojT}) mats.push_back(m);
      mats.push_back(&T->proj);
      mats.push_back(&T->projT);
    }
    for (Mat* m : mats) {
      if (!m->packed) MMX_TRY(dalloc(h, &m->packed, pack_f16x3_bytes(m->N, m->K)));
      MMX_TRY(pack_f16x3(m->w, m->K, m->N, m->K, m->packed, st));
    }
  }
  MMX_CHECK_CUDA(cudaStreamSynchronize(st));
  h->finalized = true;
  return 0;
}

int mmx_clip_interpret_device(mmx_clip* h, const float* images, int n_images, const int32_t* tokens, int B, int start_layer,
                              int start_layer_text, float* R_text, float* R_image, void* stream) {
  MMX_REQUIRE(h && h->finalized, "engine not finalized");
  MMX_REQUIRE(B > 0 && (n_images == B || n_images == 1), "n_images must be B or 1");
  int sv = 0, stx = 0;
  MMX_TRY(resolve_start(start_layer, h->v.L, &sv));
  MMX_TRY(resolve_start(start_layer_text, h->t.L, &stx));
  // NULL is the legacy default stream, like everywhere else in this ABI: the towers fork from it (so they are ordered
  // after whatever the caller enqueued there - an H2D copy, a collective that produced the inputs) and join it again.
  // (Through round 2 a NULL stream meant the engine's own non-blocking stream, which does NOT wait for default-stream
  // work: inputs still in flight on the default stream were read too early - found by bench.py's sharded == single check.)
  cudaStream_t caller = (cudaStream_t)stream;
  const size_t img_sz = (size_t)3 * h->cfg.image_resolution * h->cfg.image_resolution;
  for (int b0 = 0; b0 < B; b0 += h->Bm) {
    const int nb = (B - b0 < h->Bm) ? B - b0 : h->Bm;
    const float* img = (n_images == 1) ? images : images + (size_t)b0 * img_sz;
    MMX_TRY(run_chunk(h, img, n_images == 1 ? 1 : nb, tokens + (size_t)b0 * h->t.S, nb, sv, stx,
                      R_text + (size_t)b0 * h->t.S * h->t.S, R_image + (size_t)b0 * (h->v.S - 1), caller));
    if (b0 == 0) { h->lastB = nb; h->last_start_v = sv; h->last_start_t = stx; }
  }
  return 0;
}

int mmx_clip_interpret_host(mmx_clip* h, const float* images, int n_images, const int32_t* tokens, int B, int start_layer,
                            int start_layer_text, float* R_text, float* R_image) {
  MMX_REQUIRE(h && h->finalized, "engine not finalized");
  MMX_REQUIRE(B > 0 && (n_images == B || n_images == 1), "n_images must be B or 1");
  const size_t img_sz = (size_t)3 * h->cfg.image_resolution * h->cfg.image_resolution;
  const int St = h->t.S, Sv = h->v.S;
  cudaStream_t st = h->main;
  for (int b0 = 0; b0 < B; b0 += h->Bm) {
    const int nb = (B - b0 < h->Bm) ? B - b0 : h->Bm;
    const int ni = (n_images == 1) ? 1 : nb;
    const float* img = (n_images == 1) ? images : images + (size_t)b0 * img_sz;
    // The images (38.5 MB for 64 x 3 x 224^2) go up on the VISION stream: run_chunk forks both tower streams from `st`,
    // so the text tower starts as soon as the tokens are there and runs under the image copy; the vision tower follows
    // its own stream's copy.  (The previous chunk ended with a synchronise on `st` after joining both towers.)
    if (n_images != 1 || b0 == 0)
      MMX_CHECK_CUDA(cudaMemcpyAsync(h->d_images, img, ni * img_sz * sizeof(float), cudaMemcpyHostToDevice, h->v.st));
    MMX_CHECK_CUDA(cudaMemcpyAsync(h->d_tokens, tokens + (size_t)b0 * St, (size_t)nb * St * sizeof(int32_t),
                                   cudaMemcpyHostToDevice, st));
    MMX_TRY(mmx_clip_interpret_device(h, h->d_images, ni, h->d_tokens, nb, start_layer, start_layer_text, h->d_Rtext,
                                      h->d_Rimage, st));
    MMX_CHECK_CUDA(cudaMemcpyAsync(R_text + (size_t)b0 * St * St, h->d_Rtext, (size_t)nb * St * St * sizeof(float),
                                   cudaMemcpyDeviceToHost, st));
    MMX_CHECK_CUDA(cudaMemcpyAsync(R_image + (size_t)b0 * (Sv - 1), h->d_Rimage, (size_t)nb * (Sv - 1) * sizeof(float),
                                   cudaMemcpyDeviceToHost, st));
    MMX_CHECK_CUDA(cudaStreamSynchronize(st));
  }
  return 0;
}

int mmx_clip_tap(mmx_clip* h, const char* what, int tower, int layer, const float** ptr, int dims[4], int* ld) {
  MMX_REQUIRE(h && what && ptr && dims && ld, "bad arguments");
  MMX_REQUIRE(h->lastB > 0, "no interpret call yet");
  const std::string w(what);
  const int B = h->lastB;
  if (w == "logits") {
    *ptr = h->logits; dims[0] = B; dims[1] = B; dims[2] = dims[3] = 1; *ld = B;
    return 0;
  }
  MMX_REQUIRE(tower == 0 || tower == 1, "tower must be 0 (vision) or 1 (text)");
  Tower& T = tower == 0 ? h->v : h->t;
  const int E = h->E;
  if (w == "feat" || w == "featn" || w == "dfeat") {
    *ptr = w == "feat" ? T.feat : (w == "featn" ? T.featn : T.dfeat);
    dims[0] = B; dims[1] = E; dims[2] = dims[3] = 1; *ld = E;
    return 0;
  }
  if (w == "gscale") {
    *ptr = T.gscale; dims[0] = B; dims[1] = dims[2] = dims[3] = 1; *ld = B;
    return 0;
  }
  // activation arena: layer stride B*S rows; a ragged tower's live rows are the first rows_host of each layer
  const size_t M = (size_t)T.M(B), MD = M * T.D;
  const int rows = (T.ragged && T.rows_host >= 0) ? T.rows_host : (int)M;
  if (w == "x") {
    MMX_REQUIRE(layer >= 0 && layer <= T.L, "layer out of range");
    *ptr = T.x + layer * MD; dims[0] = rows; dims[1] = T.D; dims[2] = dims[3] = 1; *ld = T.D;
    return 0;
  }
  MMX_REQUIRE(layer >= 0 && layer < T.L, "layer out of range");
  if (w == "xmid" || w == "qkv" || w == "f") {
    const int n = w == "xmid" ? 1 : (w == "qkv" ? 3 : 4);
    *ptr = (w == "xmid" ? T.xmid : (w == "qkv" ? T.qkv : T.f)) + layer * MD * n;
    dims[0] = rows; dims[1] = n * T.D; dims[2] = dims[3] = 1; *ld = n * T.D;
    return 0;
  }
  if (w == "stats") {
    *ptr = T.stats + (size_t)layer * 4 * M; dims[0] = 4; dims[1] = rows; dims[2] = dims[3] = 1; *ld = (int)M;
    return 0;
  }
  const size_t plane = (size_t)B * T.H * T.S * T.ld;
  if (w == "A" || w == "dA") {
    *ptr = (w == "A" ? T.A : T.dA) + layer * plane;
    dims[0] = B; dims[1] = T.H; dims[2] = T.S; dims[3] = T.S; *ld = T.ld;
    return 0;
  }
  if (w == "Abar") {
    *ptr = T.Abar + layer * (size_t)B * T.S * T.ld;
    dims[0] = B; dims[1] = T.S; dims[2] = T.S; dims[3] = 1; *ld = T.ld;
    return 0;
  }
  MMX_REQUIRE(false, "unknown tap");
  return 2;
}

}  // extern "C"
