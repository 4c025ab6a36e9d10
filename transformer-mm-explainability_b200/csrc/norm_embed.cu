// Row-wise kernels around the GEMMs: LayerNorm forward/backward (one warp per row), CLIP token assembly
// (patch im2col, class/positional embedding, token embedding) and the logit head with its analytic backward.
#include "mmx_common.cuh"
#include <math_constants.h>
#include <initializer_list>

namespace mmx {

// ------------------------------------------------------------------ LayerNorm
__global__ void __launch_bounds__(256) layernorm_fwd_kernel(const float* __restrict__ x, int ldx,
                                                            const int* __restrict__ row_map,
                                                            const float* __restrict__ gamma, const float* __restrict__ beta,
                                                            float* __restrict__ y, int ldy, float* __restrict__ mean,
                                                            float* __restrict__ rstd, int rows, int D, float eps,
                                                            const int* __restrict__ rows_dev) {
  const int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (rows_dev) rows = min(rows, __ldg(rows_dev));
  if (r >= rows) return;
  const float* xr = x + (long long)(row_map ? row_map[r] : r) * ldx;
  float s = 0.f;
  for (int i = lane; i < D; i += 32) s += xr[i];
  const float mu = warp_sum(s) / (float)D;
  float v = 0.f;
  for (int i = lane; i < D; i += 32) { const float d = xr[i] - mu; v = fmaf(d, d, v); }
  const float rs = rsqrtf(warp_sum(v) / (float)D + eps);
  float* yr = y + (long long)r * ldy;
  for (int i = lane; i < D; i += 32) yr[i] = (xr[i] - mu) * rs * gamma[i] + beta[i];
  if (lane == 0) {
    if (mean) mean[r] = mu;
    if (rstd) rstd[r] = rs;
  }
}

// dx = rstd * (g*dy - mean(g*dy) - xhat * mean(g*dy*xhat)) (+ residual_grad)
__global__ void __launch_bounds__(256) layernorm_bwd_kernel(const float* __restrict__ dy, int lddy,
                                                            const float* __restrict__ x, int ldx,
                                                            const int* __restrict__ row_map,
                                                            const float* __restrict__ gamma, const float* __restrict__ mean,
                                                            const float* __restrict__ rstd,
                                                            const float* __restrict__ resid, int ldres,
                                                            float* __restrict__ dx, int lddx, int rows, int D,
                                                            const int* __restrict__ rows_dev) {
  const int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (rows_dev) rows = min(rows, __ldg(rows_dev));
  if (r >= rows) return;
  const long long xrow = row_map ? row_map[r] : r;
  const float* xr = x + xrow * ldx;
  const float* dyr = dy + (long long)r * lddy;
  const float mu = mean[r], rs = rstd[r];
  float s1 = 0.f, s2 = 0.f;
  for (int i = lane; i < D; i += 32) {
    const float g = gamma[i] * dyr[i];
    s1 += g;
    s2 = fmaf(g, (xr[i] - mu) * rs, s2);
  }
  s1 = warp_sum(s1) / (float)D;
  s2 = warp_sum(s2) / (float)D;
  float* dxr = dx + xrow * lddx;
  const float* rr = resid ? resid + xrow * ldres : nullptr;
  for (int i = lane; i < D; i += 32) {
    const float g = gamma[i] * dyr[i];
    float v = rs * (g - s1 - (xr[i] - mu) * rs * s2);
    if (rr) v += rr[i];
    dxr[i] = v;
  }
}

// Register-cached variants: one warp per row, the row (D <= 1024, D % 128 == 0) is read ONCE as 128-bit loads and kept
// in registers across the mean / variance / output passes (2 reads + 1 write of HBM traffic total per LN forward).
template <int NV>   // NV = D / 128 float4 per lane
__global__ void __launch_bounds__(256) layernorm_fwd_vec_kernel(const float* __restrict__ x, int ldx,
                                                                const int* __restrict__ row_map,
                                                                const float* __restrict__ gamma, const float* __restrict__ beta,
                                                                float* __restrict__ y, int ldy, float* __restrict__ mean,
                                                                float* __restrict__ rstd, int rows, float eps,
                                                                const int* __restrict__ rows_dev) {
  constexpr int D = NV * 128;
  const int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  pdl_wait();                                          // launched as a programmatic dependent (launch_pdl)
  if (rows_dev) rows = min(rows, __ldg(rows_dev));
  if (r >= rows) return;
  const float4* xr = reinterpret_cast<const float4*>(x + (long long)(row_map ? row_map[r] : r) * ldx);
  float4 v[NV];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) { v[i] = xr[lane + 32 * i]; s += (v[i].x + v[i].y) + (v[i].z + v[i].w); }
  const float mu = warp_sum(s) / (float)D;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const float a = v[i].x - mu, b = v[i].y - mu, c = v[i].z - mu, d = v[i].w - mu;
    q = fmaf(a, a, q); q = fmaf(b, b, q); q = fmaf(c, c, q); q = fmaf(d, d, q);
  }
  const float rs = rsqrtf(warp_sum(q) / (float)D + eps);
  float4* yr = reinterpret_cast<float4*>(y + (long long)r * ldy);
  const float4* g4 = reinterpret_cast<const float4*>(gamma);
  const float4* b4 = reinterpret_cast<const float4*>(beta);
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const float4 g = g4[lane + 32 * i], b = b4[lane + 32 * i];
    float4 o;
    o.x = (v[i].x - mu) * rs * g.x + b.x; o.y = (v[i].y - mu) * rs * g.y + b.y;
    o.z = (v[i].z - mu) * rs * g.z + b.z; o.w = (v[i].w - mu) * rs * g.w + b.w;
    yr[lane + 32 * i] = o;
  }
  if (lane == 0) {
    if (mean) mean[r] = mu;
    if (rstd) rstd[r] = rs;
  }
}

template <int NV>
__global__ void __launch_bounds__(256) layernorm_bwd_vec_kernel(const float* __restrict__ dy, int lddy,
                                                                const float* __restrict__ x, int ldx,
                                                                const int* __restrict__ row_map,
                                                                const float* __restrict__ gamma, const float* __restrict__ mean,
                                                                const float* __restrict__ rstd,
                                                                const float* __restrict__ resid, int ldres,
                                                                float* __restrict__ dx, int lddx, int rows,
                                                                const int* __restrict__ rows_dev) {
  constexpr int D = NV * 128;
  const int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  pdl_wait();                                          // launched as a programmatic dependent (launch_pdl)
  if (rows_dev) rows = min(rows, __ldg(rows_dev));
  if (r >= rows) return;
  const long long xrow = row_map ? row_map[r] : r;
  const float4* xr = reinterpret_cast<const float4*>(x + xrow * ldx);
  const float4* dyr = reinterpret_cast<const float4*>(dy + (long long)r * lddy);
  const float4* g4 = reinterpret_cast<const float4*>(gamma);
  const float mu = mean[r], rs = rstd[r];
  float4 gd[NV], xh[NV];
  float s1 = 0.f, s2 = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const float4 g = g4[lane + 32 * i], d = dyr[lane + 32 * i], xv = xr[lane + 32 * i];
    gd[i] = make_float4(g.x * d.x, g.y * d.y, g.z * d.z, g.w * d.w);
    xh[i] = make_float4((xv.x - mu) * rs, (xv.y - mu) * rs, (xv.z - mu) * rs, (xv.w - mu) * rs);
    s1 += (gd[i].x + gd[i].y) + (gd[i].z + gd[i].w);
    s2 = fmaf(gd[i].x, xh[i].x, s2); s2 = fmaf(gd[i].y, xh[i].y, s2);
    s2 = fmaf(gd[i].z, xh[i].z, s2); s2 = fmaf(gd[i].w, xh[i].w, s2);
  }
  s1 = warp_sum(s1) / (float)D;
  s2 = warp_sum(s2) / (float)D;
  float4* dxr = reinterpret_cast<float4*>(dx + xrow * lddx);
  const float4* rr = resid ? reinterpret_cast<const float4*>(resid + xrow * ldres) : nullptr;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    float4 o;
    o.x = rs * (gd[i].x - s1 - xh[i].x * s2); o.y = rs * (gd[i].y - s1 - xh[i].y * s2);
    o.z = rs * (gd[i].z - s1 - xh[i].z * s2); o.w = rs * (gd[i].w - s1 - xh[i].w * s2);
    if (rr) { const float4 q = rr[lane + 32 * i]; o.x += q.x; o.y += q.y; o.z += q.z; o.w += q.w; }
    dxr[lane + 32 * i] = o;
  }
}

static bool ln_vec_ok(int D, std::initializer_list<const void*> ptrs, std::initializer_list<int> lds) {
  if (D % 128 != 0 || D > 1024) return false;
  for (const void* p : ptrs) if (p != nullptr && !aligned16(p)) return false;
  for (int ld : lds) if (ld % 4 != 0) return false;
  return true;
}

int layernorm_fwd(const float* x, int ldx, const int* row_map, const float* gamma, const float* beta, float* y, int ldy,
                  float* mean, float* rstd, int rows, int D, float eps, cudaStream_t st, const int* rows_dev) {
  if (rows == 0) return 0;
  if (ln_vec_ok(D, {x, gamma, beta, y}, {ldx, ldy})) {
    const int g = cdiv(rows, 8);
#define MMX_LN_F(NV) MMX_CHECK_CUDA(launch_pdl(layernorm_fwd_vec_kernel<NV>, dim3(g), dim3(256), 0, st, x, ldx, row_map, gamma, beta, y, ldy, mean, rstd, rows, eps, rows_dev))
    switch (D / 128) {
      case 1: MMX_LN_F(1); break; case 2: MMX_LN_F(2); break; case 3: MMX_LN_F(3); break; case 4: MMX_LN_F(4); break;
      case 5: MMX_LN_F(5); break; case 6: MMX_LN_F(6); break; case 7: MMX_LN_F(7); break; default: MMX_LN_F(8); break;
    }
#undef MMX_LN_F
    MMX_LAUNCH_CHECK();
    return 0;
  }
  layernorm_fwd_kernel<<<cdiv(rows, 8), 256, 0, st>>>(x, ldx, row_map, gamma, beta, y, ldy, mean, rstd, rows, D, eps, rows_dev);
  MMX_LAUNCH_CHECK();
  return 0;
}
int layernorm_bwd(const float* dy, int lddy, const float* x, int ldx, const int* row_map, const float* gamma,
                  const float* mean, const float* rstd, const float* resid, int ldres, float* dx, int lddx, int rows, int D,
                  cudaStream_t st, const int* rows_dev) {
  if (rows == 0) return 0;
  if (ln_vec_ok(D, {dy, x, gamma, resid, dx}, {lddy, ldx, lddx, resid ? ldres : 0})) {
    const int g = cdiv(rows, 8);
#define MMX_LN_B(NV) MMX_CHECK_CUDA(launch_pdl(layernorm_bwd_vec_kernel<NV>, dim3(g), dim3(256), 0, st, dy, lddy, x, ldx, row_map, gamma, mean, rstd, resid, ldres, dx, lddx, rows, rows_dev))
    switch (D / 128) {
      case 1: MMX_LN_B(1); break; case 2: MMX_LN_B(2); break; case 3: MMX_LN_B(3); break; case 4: MMX_LN_B(4); break;
      case 5: MMX_LN_B(5); break; case 6: MMX_LN_B(6); break; case 7: MMX_LN_B(7); break; default: MMX_LN_B(8); break;
    }
#undef MMX_LN_B
    MMX_LAUNCH_CHECK();
    return 0;
  }
  layernorm_bwd_kernel<<<cdiv(rows, 8), 256, 0, st>>>(dy, lddy, x, ldx, row_map, gamma, mean, rstd, resid, ldres, dx, lddx,
                                                      rows, D, rows_dev);
  MMX_LAUNCH_CHECK();
  return 0;
}

// ------------------------------------------------------------------ CLIP vision tokens
// images [n_img,3,R,R] -> patches [n_img*G*G, 3*p*p] in conv-weight order (c, i, j)  (CLIP/clip/model.py:230-232)
__global__ void __launch_bounds__(256) im2col_patch_kernel(const float* __restrict__ img, float* __restrict__ out, int n_img,
                                                           int R, int p, int G) {
  const int K = 3 * p * p;
  const long long total = (long long)n_img * G * G * K / 4;   // p % 4 == 0 -> float4 along j
  for (long long it = (long long)blockIdx.x * blockDim.x + threadIdx.x; it < total; it += (long long)gridDim.x * blockDim.x) {
    const long long e = it * 4;
    const int k = (int)(e % K);
    const long long row = e / K;
    const int gx = (int)(row % G), gy = (int)((row / G) % G);
    const long long n = row / ((long long)G * G);
    const int j = k % p, i = (k / p) % p, c = k / (p * p);
    const float* src = img + ((n * 3 + c) * R + (gy * p + i)) * (long long)R + gx * p + j;
    *reinterpret_cast<float4*>(out + e) = *reinterpret_cast<const float4*>(src);
  }
}
__global__ void __launch_bounds__(256) im2col_patch_scalar_kernel(const float* __restrict__ img, float* __restrict__ out,
                                                                  int n_img, int R, int p, int G) {
  const int K = 3 * p * p;
  const long long total = (long long)n_img * G * G * K;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int k = (int)(e % K);
    const long long row = e / K;
    const int gx = (int)(row % G), gy = (int)((row / G) % G);
    const long long n = row / ((long long)G * G);
    const int j = k % p, i = (k / p) % p, c = k / (p * p);
    out[e] = img[((n * 3 + c) * R + (gy * p + i)) * (long long)R + gx * p + j];
  }
}

// x[b,0,:] = cls + pos[0];  x[b,1+g,:] = patch_emb[(b % n_img)*G*G + g,:] + pos[1+g]  (CLIP/clip/model.py:233-234),
// one warp per token row; the ln_pre that follows (:235) is fused: writes LN(x) only.
__global__ void __launch_bounds__(256) vision_tokens_lnpre_kernel(const float* __restrict__ patch_emb, int n_img,
                                                                  const float* __restrict__ cls, const float* __restrict__ pos,
                                                                  const float* __restrict__ gamma, const float* __restrict__ beta,
                                                                  float* __restrict__ x, int B, int S, int D, float eps) {
  const int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (r >= B * S) return;
  const int b = r / S, s = r % S;
  const float* src = (s == 0) ? cls : patch_emb + ((long long)(b % n_img) * (S - 1) + (s - 1)) * D;
  const float* pr = pos + (long long)s * D;
  float sum = 0.f;
  for (int i = lane; i < D; i += 32) sum += src[i] + pr[i];
  const float mu = warp_sum(sum) / (float)D;
  float v = 0.f;
  for (int i = lane; i < D; i += 32) { const float d = src[i] + pr[i] - mu; v = fmaf(d, d, v); }
  const float rs = rsqrtf(warp_sum(v) / (float)D + eps);
  float* xr = x + (long long)r * D;
  for (int i = lane; i < D; i += 32) xr[i] = (src[i] + pr[i] - mu) * rs * gamma[i] + beta[i];
}

// text: x[b,s,:] = tok_emb[tokens[b,s]] + pos[s]   (CLIP/clip/model.py:350-352); eot[b] = first argmax_s tokens[b,s] (:360)
__global__ void __launch_bounds__(256) text_embed_kernel(const int* __restrict__ tokens, const float* __restrict__ emb,
                                                         const float* __restrict__ pos, float* __restrict__ x,
                                                         int* __restrict__ eot_row, int B, int S, int D, int vocab) {
  const int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (r >= B * S) return;
  const int b = r / S, s = r % S;
  int tok = tokens[r];
  tok = tok < 0 ? 0 : (tok >= vocab ? vocab - 1 : tok);
  const float* er = emb + (long long)tok * D;
  const float* pr = pos + (long long)s * D;
  float* xr = x + (long long)r * D;
  for (int i = lane; i < D; i += 32) xr[i] = er[i] + pr[i];
  if (s == 0) {
    int best = -2147483647 - 1, bi = 0;
    for (int j = lane; j < S; j += 32) {
      const int t = tokens[b * S + j];
      if (t > best) { best = t; bi = j; }
    }
    for (int o = 16; o > 0; o >>= 1) {
      const int ob = __shfl_xor_sync(0xffffffffu, best, o), oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
    }
    if (lane == 0) eot_row[b] = b * S + bi;
  }
}

// Ragged text batches.  Under the causal mask a token never sees later tokens and only the EOT feature is pooled
// (CLIP/clip/model.py:334-340,360), so rows after the EOT cannot influence the logits; the reference still computes
// them (their A rows get zero gradient, their R rows stay identity).  lens[b] = eot_b + 1 rows per sample are kept,
// packed back to back: offs = exclusive scan, total = sum, eot_row[b] = offs[b] + lens[b] - 1.
__global__ void __launch_bounds__(256) text_lens_kernel(const int* __restrict__ tokens, int* __restrict__ lens, int B, int S) {
  const int b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (b >= B) return;
  int best = -2147483647 - 1, bi = 0;
  for (int j = lane; j < S; j += 32) {
    const int t = tokens[b * S + j];
    if (t > best) { best = t; bi = j; }
  }
  for (int o = 16; o > 0; o >>= 1) {
    const int ob = __shfl_xor_sync(0xffffffffu, best, o), oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
  }
  if (lane == 0) lens[b] = bi + 1;
}
__global__ void text_scan_kernel(const int* __restrict__ lens, int* __restrict__ offs, int* __restrict__ eot_row,
                                 int* __restrict__ total, int B) {
  if (blockIdx.x != 0 || threadIdx.x != 0) return;     // B is a batch size (<= a few thousand): a serial scan is free
  int acc = 0;
  for (int b = 0; b < B; ++b) {
    offs[b] = acc;
    acc += lens[b];
    eot_row[b] = acc - 1;
  }
  *total = acc;
}
__global__ void __launch_bounds__(256) text_embed_packed_kernel(const int* __restrict__ tokens, const float* __restrict__ emb,
                                                                const float* __restrict__ pos, float* __restrict__ x,
                                                                const int* __restrict__ offs, const int* __restrict__ lens,
                                                                int B, int S, int D, int vocab) {
  const int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (r >= B * S) return;
  const int b = r / S, sidx = r % S;
  if (sidx >= lens[b]) return;
  int tok = tokens[r];
  tok = tok < 0 ? 0 : (tok >= vocab ? vocab - 1 : tok);
  const float* er = emb + (long long)tok * D;
  const float* pr = pos + (long long)sidx * D;
  float* xr = x + (long long)(offs[b] + sidx) * D;
  for (int i = lane; i < D; i += 32) xr[i] = er[i] + pr[i];
}

__global__ void cls_rows_kernel(int* __restrict__ rows, int B, int S) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b < B) rows[b] = b * S;
}

// logits head (CLIP/clip/model.py:368-374) and its analytic backward for y = sum_b logits[b,b]
// (CLIP_explainability.ipynb:156-160).  One warp per sample.
//   fi_n = fi/|fi|, ft_n = ft/|ft|, c = <fi_n, ft_n>, logit = s*c,
//   d fi = s/|fi| * (ft_n - c*fi_n),  d ft = s/|ft| * (fi_n - c*ft_n)
__global__ void __launch_bounds__(256) clip_head_kernel(const float* __restrict__ fi, const float* __restrict__ ft,
                                                        float logit_scale_exp, float* __restrict__ fin,
                                                        float* __restrict__ ftn, float* __restrict__ dfi,
                                                        float* __restrict__ dft, float* __restrict__ diag,
                                                        float* __restrict__ gs_i, float* __restrict__ gs_t, int B, int E) {
  const int b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (b >= B) return;
  const float* a = fi + (long long)b * E;
  const float* t = ft + (long long)b * E;
  float sa = 0.f, stt = 0.f;
  for (int i = lane; i < E; i += 32) { sa = fmaf(a[i], a[i], sa); stt = fmaf(t[i], t[i], stt); }
  const float na = sqrtf(warp_sum(sa)), nt = sqrtf(warp_sum(stt));
  float c = 0.f;
  for (int i = lane; i < E; i += 32) c = fmaf(a[i] / na, t[i] / nt, c);
  c = warp_sum(c);
  float mi = 0.f, mt = 0.f;
  for (int i = lane; i < E; i += 32) {
    const float an = a[i] / na, tn = t[i] / nt;
    fin[(long long)b * E + i] = an;
    ftn[(long long)b * E + i] = tn;
    const float gi = logit_scale_exp / na * (tn - c * an), gt = logit_scale_exp / nt * (an - c * tn);
    dfi[(long long)b * E + i] = gi;
    dft[(long long)b * E + i] = gt;
    mi = fmaxf(mi, fabsf(gi)); mt = fmaxf(mt, fabsf(gt));
  }
  if (gs_i) {
    // Per-sample power-of-two normalisation of the seed gradient (max |d feat| -> [16, 32)): the fp16x3 GEMMs of the
    // dgrad sweep then see magnitudes inside fp16's range whatever the model's logit scale / feature norm is; the
    // attention backward divides the staged dA by the same factor.  Exact (powers of two) and per sample.
    mi = warp_max(mi); mt = warp_max(mt);
    const float si = (mi > 0.f && mi < CUDART_INF_F) ? exp2f(4.f - (float)ilogbf(mi)) : 1.f;
    const float st2 = (mt > 0.f && mt < CUDART_INF_F) ? exp2f(4.f - (float)ilogbf(mt)) : 1.f;
    __syncwarp();
    for (int i = lane; i < E; i += 32) { dfi[(long long)b * E + i] *= si; dft[(long long)b * E + i] *= st2; }
    if (lane == 0) { gs_i[b] = si; gs_t[b] = st2; }
  }
  if (lane == 0 && diag) diag[b] = logit_scale_exp * c;
}

__global__ void scale_kernel(float* __restrict__ x, long long n, float s) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) x[i] *= s;
}

// R[b] = I (S x S, row stride ld, pads zero)
__global__ void __launch_bounds__(256) eye_kernel(float* __restrict__ R, int B, int S, int ld) {
  const long long n = (long long)B * S * ld;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % ld);
    const int r = (int)((i / ld) % S);
    R[i] = (c == r) ? 1.f : 0.f;
  }
}

// strided copy-out: dst[b, r, c] (dense rows x cols) = src[b, r0 + r, c0 + c] (row stride ld, plane stride plane)
__global__ void __launch_bounds__(256) slice_out_kernel(const float* __restrict__ src, long long plane, int ld, int r0, int c0,
                                                        float* __restrict__ dst, int B, int rows, int cols) {
  const long long n = (long long)B * rows * cols;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % cols);
    const int r = (int)((i / cols) % rows);
    const long long b = i / ((long long)cols * rows);
    dst[i] = src[b * plane + (long long)(r0 + r) * ld + c0 + c];
  }
}

__global__ void __launch_bounds__(256) add_kernel(const float* __restrict__ a, int lda, const float* __restrict__ b, int ldb,
                                                   float alpha, float* __restrict__ out, int ldo, long long rows, int cols) {
  const long long n = rows * cols;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / cols;
    const int c = (int)(i - r * cols);
    out[r * ldo + c] = a[r * lda + c] + alpha * b[r * ldb + c];
  }
}
__global__ void __launch_bounds__(256) gather_rows_kernel(const float* __restrict__ src, int lds, const int* __restrict__ map,
                                                          float* __restrict__ out, int ldo, int rows, int cols, int scatter_add) {
  const long long n = (long long)rows * cols;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(i / cols), c = (int)(i % cols);
    if (scatter_add) out[(long long)map[r] * ldo + c] += src[(long long)r * lds + c];
    else out[(long long)r * ldo + c] = src[(long long)map[r] * lds + c];
  }
}
__global__ void __launch_bounds__(256) act_kernel(const float* __restrict__ dy, int lddy, const float* __restrict__ pre, int ldpre,
                                                  int act, float* __restrict__ out, int ldo, long long rows, int cols, int bwd) {
  const long long n = rows * cols;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / cols;
    const int c = (int)(i - r * cols);
    const float x = pre[r * ldpre + c];
    out[r * ldo + c] = bwd ? dy[r * lddy + c] * act_bwd(x, act) : act_fwd(x, act);
  }
}

static int grid_for(long long items) {
  long long g = (items + 255) / 256, cap = (long long)sm_count() * 8;
  return (int)(g > cap ? cap : (g < 1 ? 1 : g));
}

int im2col_patches(const float* img, float* out, int n_img, int R, int p, cudaStream_t st) {
  const int G = R / p;
  const long long total = (long long)n_img * G * G * 3 * p * p;
  if (total == 0) return 0;
  if (p % 4 == 0 && R % 4 == 0 && aligned16(img) && aligned16(out))
    im2col_patch_kernel<<<grid_for(total / 4), 256, 0, st>>>(img, out, n_img, R, p, G);
  else
    im2col_patch_scalar_kernel<<<grid_for(total), 256, 0, st>>>(img, out, n_img, R, p, G);
  MMX_LAUNCH_CHECK();
  return 0;
}
int vision_tokens_lnpre(const float* patch_emb, int n_img, const float* cls, const float* pos, const float* gamma,
                        const float* beta, float* x, int B, int S, int D, float eps, cudaStream_t st) {
  vision_tokens_lnpre_kernel<<<cdiv(B * S, 8), 256, 0, st>>>(patch_emb, n_img, cls, pos, gamma, beta, x, B, S, D, eps);
  MMX_LAUNCH_CHECK();
  return 0;
}
int text_embed(const int* tokens, const float* emb, const float* pos, float* x, int* eot_row, int B, int S, int D, int vocab,
               cudaStream_t st) {
  text_embed_kernel<<<cdiv(B * S, 8), 256, 0, st>>>(tokens, emb, pos, x, eot_row, B, S, D, vocab);
  MMX_LAUNCH_CHECK();
  return 0;
}
int text_embed_packed(const int* tokens, const float* emb, const float* pos, float* x, int* offs, int* lens, int* eot_row,
                      int* total, int B, int S, int D, int vocab, cudaStream_t st) {
  text_lens_kernel<<<cdiv(B, 8), 256, 0, st>>>(tokens, lens, B, S);
  MMX_LAUNCH_CHECK();
  text_scan_kernel<<<1, 32, 0, st>>>(lens, offs, eot_row, total, B);
  MMX_LAUNCH_CHECK();
  text_embed_packed_kernel<<<cdiv(B * S, 8), 256, 0, st>>>(tokens, emb, pos, x, offs, lens, B, S, D, vocab);
  MMX_LAUNCH_CHECK();
  return 0;
}
int cls_rows(int* rows, int B, int S, cudaStream_t st) {
  cls_rows_kernel<<<cdiv(B, 128), 128, 0, st>>>(rows, B, S);
  MMX_LAUNCH_CHECK();
  return 0;
}
int clip_head(const float* fi, const float* ft, float lse, float* fin, float* ftn, float* dfi, float* dft, float* diag,
              float* gs_i, float* gs_t, int B, int E, cudaStream_t st) {
  clip_head_kernel<<<cdiv(B, 8), 256, 0, st>>>(fi, ft, lse, fin, ftn, dfi, dft, diag, gs_i, gs_t, B, E);
  MMX_LAUNCH_CHECK();
  return 0;
}
int scale_inplace(float* x, long long n, float s, cudaStream_t st) {
  scale_kernel<<<grid_for(n), 256, 0, st>>>(x, n, s);
  MMX_LAUNCH_CHECK();
  return 0;
}
int set_eye(float* R, int B, int S, int ld, cudaStream_t st) {
  eye_kernel<<<grid_for((long long)B * S * ld), 256, 0, st>>>(R, B, S, ld);
  MMX_LAUNCH_CHECK();
  return 0;
}
int slice_out(const float* src, long long plane, int ld, int r0, int c0, float* dst, int B, int rows, int cols,
              cudaStream_t st) {
  slice_out_kernel<<<grid_for((long long)B * rows * cols), 256, 0, st>>>(src, plane, ld, r0, c0, dst, B, rows, cols);
  MMX_LAUNCH_CHECK();
  return 0;
}

}  // namespace mmx

using namespace mmx;
extern "C" {
int mmx_add(const float* a, int lda, const float* b, int ldb, float alpha, float* out, int ldo, long long rows, int cols,
            void* stream) {
  if (rows == 0 || cols == 0) return 0;
  add_kernel<<<grid_for(rows * cols), 256, 0, (cudaStream_t)stream>>>(a, lda, b, ldb, alpha, out, ldo, rows, cols);
  MMX_LAUNCH_CHECK();
  return 0;
}
int mmx_gather_rows(const float* src, int lds, const int32_t* row_map, float* out, int ldo, int rows, int cols, void* stream) {
  if (rows == 0 || cols == 0) return 0;
  gather_rows_kernel<<<grid_for((long long)rows * cols), 256, 0, (cudaStream_t)stream>>>(src, lds, row_map, out, ldo, rows, cols, 0);
  MMX_LAUNCH_CHECK();
  return 0;
}
int mmx_scatter_add_rows(const float* src, int lds, const int32_t* row_map, float* dst, int ldd, int rows, int cols,
                         void* stream) {
  if (rows == 0 || cols == 0) return 0;
  gather_rows_kernel<<<grid_for((long long)rows * cols), 256, 0, (cudaStream_t)stream>>>(src, lds, row_map, dst, ldd, rows, cols, 1);
  MMX_LAUNCH_CHECK();
  return 0;
}
int mmx_act_bwd(const float* dy, int lddy, const float* pre, int ldpre, int act, float* dx, int lddx, long long rows, int cols,
                void* stream) {
  if (rows == 0 || cols == 0) return 0;
  act_kernel<<<grid_for(rows * cols), 256, 0, (cudaStream_t)stream>>>(dy, lddy, pre, ldpre, act, dx, lddx, rows, cols, 1);
  MMX_LAUNCH_CHECK();
  return 0;
}
int mmx_act_fwd(const float* x, int ldx, int act, float* y, int ldy, long long rows, int cols, void* stream) {
  if (rows == 0 || cols == 0) return 0;
  act_kernel<<<grid_for(rows * cols), 256, 0, (cudaStream_t)stream>>>(nullptr, 0, x, ldx, act, y, ldy, rows, cols, 0);
  MMX_LAUNCH_CHECK();
  return 0;
}
int mmx_im2col_patches(const float* images, float* patches, int n_images, int resolution, int patch, void* stream) {
  MMX_REQUIRE(patch > 0 && resolution % patch == 0, "resolution must be a multiple of patch");
  return im2col_patches(images, patches, n_images, resolution, patch, (cudaStream_t)stream);
}
int mmx_layernorm_fwd(const float* x, int ldx, const int* row_map, const float* gamma, const float* beta, float* y, int ldy,
                      float* mean, float* rstd, int rows, int D, float eps, void* stream) {
  return layernorm_fwd(x, ldx, row_map, gamma, beta, y, ldy, mean, rstd, rows, D, eps, (cudaStream_t)stream, nullptr);
}
int mmx_layernorm_bwd(const float* dy, int lddy, const float* x, int ldx, const int* row_map, const float* gamma,
                      const float* mean, const float* rstd, const float* residual_grad, int ldres, float* dx, int lddx,
                      int rows, int D, void* stream) {
  return layernorm_bwd(dy, lddy, x, ldx, row_map, gamma, mean, rstd, residual_grad, ldres, dx, lddx, rows, D,
                       (cudaStream_t)stream, nullptr);
}
int mmx_text_embed_packed(const int32_t* tokens, const float* emb, const float* pos, float* x, int* offs, int* lens,
                          int* eot_row, int* total, int B, int S, int D, int vocab, void* stream) {
  MMX_REQUIRE(B > 0 && S > 0 && D > 0 && vocab > 0, "bad sizes");
  return text_embed_packed(tokens, emb, pos, x, offs, lens, eot_row, total, B, S, D, vocab, (cudaStream_t)stream);
}
int mmx_vision_tokens_lnpre(const float* patch_emb, int n_img, const float* cls, const float* pos, const float* gamma,
                            const float* beta, float* x, int B, int S, int D, float eps, void* stream) {
  MMX_REQUIRE(B > 0 && S > 1 && D > 0 && n_img > 0, "bad sizes");
  return vision_tokens_lnpre(patch_emb, n_img, cls, pos, gamma, beta, x, B, S, D, eps, (cudaStream_t)stream);
}
int mmx_clip_head(const float* fi, const float* ft, float logit_scale_exp, float* fin, float* ftn, float* dfi, float* dft,
                  float* diag, float* gs_i, float* gs_t, int B, int E, void* stream) {
  MMX_REQUIRE(B > 0 && E > 0, "bad sizes");
  MMX_REQUIRE(fi && ft && fin && ftn && dfi && dft, "fi, ft, fin, ftn, dfi and dft are required");
  MMX_REQUIRE((gs_i == nullptr) == (gs_t == nullptr), "gs_i / gs_t: both or neither");
  return clip_head(fi, ft, logit_scale_exp, fin, ftn, dfi, dft, diag, gs_i, gs_t, B, E, (cudaStream_t)stream);
}
}
