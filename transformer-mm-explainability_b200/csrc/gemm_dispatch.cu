// GEMM backend dispatch + the exported linear / linear_dgrad entry points and library-wide state.
#include "gemm.cuh"
#include <mutex>
#include <vector>
#include <cstdlib>

namespace mmx {

static thread_local std::string g_error;
std::atomic<uint64_t> g_launches{0};
static std::atomic<int> g_backend{-1};

void set_error(const std::string& msg) { g_error = msg; }
const char* last_error() { return g_error.c_str(); }

int sm_count() {
  static std::atomic<int> n[MMX_MAX_DEVICES];   // zero-initialised; benign race: every writer stores the same value
  const int dev = current_device();
  int v = n[dev].load(std::memory_order_relaxed);
  if (v == 0) {
    if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0) v = 132;
    n[dev].store(v, std::memory_order_relaxed);
  }
  return v;
}

// gemm_wgmma.cu
bool gemm_tc_shape_ok(const float* A, int lda, const float* Bt, int ldb, float* C, int ldc, int N, int K,
                      const GemmEpilogue& ep);
int gemm_nt_tc(const float* A, int lda, const float* Bt, int ldb, float* C, int ldc, int M, int N, int K,
               const GemmEpilogue& ep, cudaStream_t st);

int gemm_nt_tc_batched(const float* A, int lda, int rows_a, const float* Bt, int ldb, int rows_b, float* C, int ldc, long long stride_c,
                       long long stride_res, int M, int N, int K, int batch, const GemmEpilogue& ep, cudaStream_t st);
void attention_set_trace(long long* buf);

int gemm_backend() {
  int b = g_backend.load();
  if (b < 0) {
    b = gemm_tc_available() ? 3 : 0;   // H100: the pre-split pass + TMA -> wgmma loop beats the in-kernel split (DESIGN.md §4.1)
    const char* env = getenv("MMX_GEMM_BACKEND");
    if (env && b) b = atoi(env) < 0 ? 0 : (atoi(env) > 3 ? 3 : atoi(env));   // 0 FFMA, 1 tf32x3, 2 fp16x3 (packed weights), 3 fp16x3 with A pre-split
    g_backend.store(b);
  }
  return b;
}

bool gemm_a_act_ok(const float* A, int lda, const BOperand& B, float* C, int ldc, int N, int K, const GemmEpilogue& ep) {
  return gemm_backend() == 3 && B.hi && gemm_f16x3_shape_ok(A, lda, B, C, ldc, N, K, ep);
}

static int gemm_nt_impl(const float* A, int lda, const BOperand& B, float* C, int ldc, int M, int N, int K,
                        const GemmEpilogue& ep, cudaStream_t st) {
  const int be = gemm_backend();
  if (ep.a_act != MMX_ACT_NONE) {
    MMX_REQUIRE(gemm_a_act_ok(A, lda, B, C, ldc, N, K, ep), "an activation on A needs the fp16x3 pre-split backend");
    return gemm_nt_f16x3(A, lda, B, C, ldc, M, N, K, ep, st, true);
  }
  if (be >= 2 && B.hi && gemm_f16x3_shape_ok(A, lda, B, C, ldc, N, K, ep)) return gemm_nt_f16x3(A, lda, B, C, ldc, M, N, K, ep, st, be == 3);
  if (be >= 1 && gemm_tc_shape_ok(A, lda, B.w, B.ldw, C, ldc, N, K, ep)) return gemm_nt_tc(A, lda, B.w, B.ldw, C, ldc, M, N, K, ep, st);
  return gemm_nt_simt(A, lda, B.w, B.ldw, C, ldc, M, N, K, ep, st);
}

int gemm_nt_tc_rule(const float* A, int lda, long long rows_a, const float* Bt, int ldb, long long rows_b, const float* residual,
                    int ldres, long long stride_res, float* C, int ldc, long long stride_c, int M, int N, int K, int batch,
                    cudaStream_t st, bool* taken) {
  *taken = false;
  const int Np = round_up(N, 4);
  if (gemm_backend() < 1 || !gemm_tc_available()) return 0;
  if (M < 128 || N < 128 || K < 64 || (lda % 4) || (ldb % 4) || (ldc % 4) || ldc < Np) return 0;
  if (residual && ((ldres % 4) || ldres < Np || !aligned16(residual) || (stride_res % 4))) return 0;
  if (!aligned16(A) || !aligned16(Bt) || !aligned16(C) || (stride_c % 4)) return 0;
  GemmEpilogue ep;
  ep.residual = residual; ep.ldres = ldres;
  *taken = true;
  // N is passed rounded up: rows N..Np-1 of Bt[b] hold the transposed pad (zeros), the pad columns of C get 0 + residual pad
  return gemm_nt_tc_batched(A, lda, (int)rows_a, Bt, ldb, (int)rows_b, C, ldc, stride_c, stride_res, M, Np, K, batch, ep, st);
}

// Optional per-launch CUDA-event timing of the GEMMs (the dominant kernel) for bench.py's roofline line.
struct ProfRec { cudaEvent_t s, e; double flops; const int* m_dev; int M; };
static std::mutex g_prof_mu;
static std::vector<ProfRec> g_prof;       // records of the current profiling window
static std::vector<cudaEvent_t> g_pool;   // reusable events
static std::atomic<int> g_prof_on{0};

int gemm_nt(const float* A, int lda, const float* Bt, int ldb, float* C, int ldc, int M, int N, int K,
            const GemmEpilogue& ep, cudaStream_t st) {
  BOperand B;
  B.w = Bt; B.ldw = ldb;
  return gemm_nt_b(A, lda, B, C, ldc, M, N, K, ep, st);
}

// run(): one GEMM launch sequence; timed by CUDA events when a profiling window is open
template <typename Run>
static int profiled(int M, int N, int K, const GemmEpilogue& ep, cudaStream_t st, Run run) {
  if (!g_prof_on.load(std::memory_order_relaxed) || M == 0 || N == 0) return run();
  ProfRec r;
  {
    std::lock_guard<std::mutex> lk(g_prof_mu);
    for (cudaEvent_t* ev : {&r.s, &r.e}) {
      if (!g_pool.empty()) { *ev = g_pool.back(); g_pool.pop_back(); }
      else MMX_CHECK_CUDA(cudaEventCreate(ev));
    }
  }
  r.flops = 2.0 * (double)M * (double)N * (double)K;
  r.m_dev = ep.m_dev;
  r.M = M;
  MMX_CHECK_CUDA(cudaEventRecord(r.s, st));
  MMX_TRY(run());
  MMX_CHECK_CUDA(cudaEventRecord(r.e, st));
  std::lock_guard<std::mutex> lk(g_prof_mu);
  g_prof.push_back(r);
  return 0;
}

int gemm_nt_b(const float* A, int lda, const BOperand& Bop, float* C, int ldc, int M, int N, int K, const GemmEpilogue& ep,
              cudaStream_t st) {
  return profiled(M, N, K, ep, st, [&] { return gemm_nt_impl(A, lda, Bop, C, ldc, M, N, K, ep, st); });
}

int gemm_nt_planes(const uint16_t* Ahi, const uint16_t* Alo, int ldpa, const BOperand& B, float* C, int ldc, int M, int N, int K,
                   const GemmEpilogue& ep, cudaStream_t st) {
  MMX_REQUIRE(ep.a_act == MMX_ACT_NONE, "an activation on A needs the fp16x3 pre-split backend");
  return profiled(M, N, K, ep, st, [&] { return gemm_nt_f16x3_planes(Ahi, Alo, ldpa, B, C, ldc, M, N, K, ep, st); });
}

}  // namespace mmx

using namespace mmx;
extern "C" {
const char* mmx_last_error(void) { return mmx::last_error(); }
int mmx_version(void) { return MMX_VERSION; }
uint64_t mmx_launch_count(void) { return g_launches.load(); }
int mmx_set_gemm_backend(int backend) {
  if (backend < 0) backend = 0;
  if (backend > 3) backend = 3;
  if (backend >= 1 && !gemm_tc_available()) backend = 0;
  g_backend.store(backend);
  return g_backend.load();
}

int mmx_get_gemm_backend(void) { return gemm_backend(); }

int mmx_set_gemm_tile_n(int bn) { return gemm_tc_tile_n(bn == 0 || bn == 128 || bn == 144 || bn == 160 ? bn : -1); }

int mmx_profile_gemm(int enable) {
  std::lock_guard<std::mutex> lk(g_prof_mu);
  if (enable) {
    for (ProfRec& r : g_prof) { g_pool.push_back(r.s); g_pool.push_back(r.e); }
    g_prof.clear();
  }
  g_prof_on.store(enable ? 1 : 0);
  return 0;
}
int mmx_profile_gemm_report(double* total_ms, double* total_flops, int* launches) {
  MMX_CHECK_CUDA(cudaDeviceSynchronize());
  std::lock_guard<std::mutex> lk(g_prof_mu);
  double ms = 0, fl = 0;
  for (ProfRec& r : g_prof) {
    float t = 0.f;
    MMX_CHECK_CUDA(cudaEventElapsedTime(&t, r.s, r.e));
    double f = r.flops;
    if (r.m_dev && r.M > 0) {           // ragged batch: count the rows actually processed, not the upper bound
      int m = r.M;
      MMX_CHECK_CUDA(cudaMemcpy(&m, r.m_dev, sizeof(int), cudaMemcpyDeviceToHost));
      f *= (double)(m < r.M ? m : r.M) / (double)r.M;
    }
    ms += t; fl += f;
  }
  if (total_ms) *total_ms = ms;
  if (total_flops) *total_flops = fl;
  if (launches) *launches = (int)g_prof.size();
  return 0;
}

int mmx_gemm_trace(long long* device_buf) {
  attention_set_trace(device_buf ? device_buf + 4096 : nullptr);   // the attention forward kernel's phases: slots 4096 .. 4102
  return 0;
}
int mmx_memcpy_d2d(void* dst, const void* src, size_t bytes, void* stream) {
  MMX_CHECK_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return 0;
}

size_t mmx_pack_weight_bytes(int N, int K) { return (N > 0 && K > 0) ? pack_f16x3_bytes(N, K) : 0; }
int mmx_pack_weight(const float* W, int ldw, int N, int K, void* packed, void* stream) {
  MMX_REQUIRE(W && packed && N > 0 && K > 0 && ldw >= K, "bad arguments");
  return pack_f16x3(W, ldw, N, K, packed, (cudaStream_t)stream);
}
int mmx_linear_packed(const float* A, int lda, const float* W, int ldw, const void* packed, const float* bias,
                      const float* residual, int ldres, float* C, int ldc, float* C_act, int act, int M, int N, int K,
                      void* stream) {
  GemmEpilogue ep;
  ep.bias = bias; ep.residual = residual; ep.ldres = ldres; ep.C_act = C_act; ep.act = act;
  return gemm_nt_b(A, lda, packed_operand(W, ldw, packed, N, K), C, ldc, M, N, K, ep, (cudaStream_t)stream);
}
int mmx_gemm_nt(const float* A, int lda, const float* Bt, int ldb, const void* packed, const float* bias, const float* pre,
                int ldpre, const float* residual, int ldres, float* C, int ldc, float* C_act, int act, int M, int N, int K,
                void* stream) {
  GemmEpilogue ep;
  ep.bias = bias; ep.pre = pre; ep.ldpre = ldpre; ep.residual = residual; ep.ldres = ldres; ep.C_act = C_act; ep.act = act;
  return gemm_nt_b(A, lda, packed_operand(Bt, ldb, packed, N, K), C, ldc, M, N, K, ep, (cudaStream_t)stream);
}
int mmx_linear(const float* A, int lda, const float* W, int ldw, const float* bias, const float* residual, int ldres, float* C,
               int ldc, float* C_act, int act, int M, int N, int K, void* stream) {
  return mmx_linear_packed(A, lda, W, ldw, nullptr, bias, residual, ldres, C, ldc, C_act, act, M, N, K, stream);
}
int mmx_linear_dgrad_packed(const float* dY, int lddy, const float* Wt, int ldwt, const void* packed_t, const float* pre,
                            int ldpre, int act, float* dX, int lddx, int M, int N, int K, void* stream) {
  GemmEpilogue ep;
  ep.pre = pre; ep.ldpre = ldpre; ep.act = act;
  // dX[M,K] = dY[M,N] * Wt[K,N]^T : an NT GEMM with "N" = K and reduction over N
  return gemm_nt_b(dY, lddy, packed_operand(Wt, ldwt, packed_t, K, N), dX, lddx, M, K, N, ep, (cudaStream_t)stream);
}
int mmx_linear_dgrad(const float* dY, int lddy, const float* Wt, int ldwt, const float* pre, int ldpre, int act, float* dX,
                     int lddx, int M, int N, int K, void* stream) {
  return mmx_linear_dgrad_packed(dY, lddy, Wt, ldwt, nullptr, pre, ldpre, act, dX, lddx, M, N, K, stream);
}
}
