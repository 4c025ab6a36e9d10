// DETR's ResNet backbone on the GEMM backends: convolution as gather + GEMM, max-pool and the mask / sine position
// embedding (DETR/models/backbone.py, DETR/models/position_encoding.py).
//
// Layout: activations are NHWC matrices [B*H*W, C] with a row stride, so a conv output is one GEMM C = A W^T with
// A = the gathered patches [B*Ho*Wo, kh*kw*C] in (ky, kx, c) order and W the OIHW weight reordered to [Cout, kh*kw*C]
// (the caller folds FrozenBatchNorm2d into W and bias).  A 1x1 stride-1 conv reads the activation itself as A.  Every
// other conv gathers A once; under backend 3 (the default) the gather writes the fp16 hi / lo' planes the wgmma kernel
// loads by TMA, so the conv pays one pass over its input instead of a gather plus the GEMM's own split pass.
#include "gemm.cuh"
#include <cuda_fp16.h>

namespace mmx {
namespace {

// The fp16x3 split of gemm_wgmma.cu (split2 / split_a_planes_kernel): hi = fp16_rn(x), lo' = fp16_rn((x - hi) * 2048).
// Bit-identical to it, so a 1x1 conv gives the same planes whether it is gathered here or split inside the GEMM call.
__device__ __forceinline__ void split_pair(float x0, float x1, uint32_t& hi, uint32_t& lo) {
  const __half2 h = __floats2half2_rn(x0, x1);
  const float2 hf = __half22float2(h);
  const __half2 l = __floats2half2_rn((x0 - hf.x) * 2048.f, (x1 - hf.y) * 2048.f);
  hi = *reinterpret_cast<const uint32_t*>(&h);
  lo = *reinterpret_cast<const uint32_t*>(&l);
}

struct ConvGeom {
  long long sN, sY, sX, sC;
  int H, W, C, Ho, Wo, kw, stride, pad, dil, M, K;
};

// Row m, columns k0 .. k0+3 of the patch matrix (zero outside the image and beyond K); tap (ky, kx) of output pixel
// (oy, ox) reads input pixel (oy stride - pad + ky dil, ox stride - pad + kx dil), as F.conv2d with dilation = dil.  VEC: C % 4 == 0, sC == 1 and
// every other stride and the base 16-byte aligned - the four columns are one float4 of one pixel.
template <bool VEC>
__device__ __forceinline__ float4 patch4(const float* __restrict__ x, const ConvGeom& g, int m, int k0) {
  const int hw = g.Ho * g.Wo, b = m / hw, r = m - b * hw, oy = r / g.Wo, ox = r - oy * g.Wo;
  const int iy0 = oy * g.stride - g.pad, ix0 = ox * g.stride - g.pad;
  const float* xb = x + b * g.sN;
  if constexpr (VEC) {
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    const int c = k0 % g.C, t = k0 / g.C, kx = t % g.kw, ky = t / g.kw, iy = iy0 + ky * g.dil, ix = ix0 + kx * g.dil;
    if (k0 < g.K && iy >= 0 && iy < g.H && ix >= 0 && ix < g.W)
      v = __ldg(reinterpret_cast<const float4*>(xb + iy * g.sY + ix * g.sX + c));
    return v;
  } else {
    float e[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int k = k0 + i, c = k % g.C, t = k / g.C, kx = t % g.kw, ky = t / g.kw, iy = iy0 + ky * g.dil, ix = ix0 + kx * g.dil;
      e[i] = (k < g.K && iy >= 0 && iy < g.H && ix >= 0 && ix < g.W) ? __ldg(xb + iy * g.sY + ix * g.sX + c * g.sC) : 0.f;
    }
    return make_float4(e[0], e[1], e[2], e[3]);
  }
}

// Patch matrix [M, ld] as fp32 (f32 != nullptr) or as fp16 hi / lo' planes; four columns per thread.  Columns K .. ld-1
// that a thread covers are written as zeros; the GEMM never reads beyond K.
template <bool VEC>
__global__ void __launch_bounds__(256) im2col_kernel(const float* __restrict__ x, ConvGeom g, int ld, float* __restrict__ f32,
                                                     __half* __restrict__ hi, __half* __restrict__ lo) {
  const int kc = (g.K + 3) / 4;
  const long long total = (long long)g.M * kc;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int m = (int)(i / kc), k0 = (int)(i % kc) * 4;
    const float4 v = patch4<VEC>(x, g, m, k0);
    const long long o = (long long)m * ld + k0;
    if (f32) {
      *reinterpret_cast<float4*>(f32 + o) = v;
    } else {
      uint2 h, l;
      split_pair(v.x, v.y, h.x, l.x);
      split_pair(v.z, v.w, h.y, l.y);
      *reinterpret_cast<uint2*>(hi + o) = h;
      *reinterpret_cast<uint2*>(lo + o) = l;
    }
  }
}

__global__ void __launch_bounds__(256) maxpool3s2_kernel(const float* __restrict__ in, int ldi, float* __restrict__ out, int ldo,
                                                         int B, int H, int W, int C, int Ho, int Wo) {
  const long long total = (long long)B * Ho * Wo * C;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const long long r = i / C;
    const int ox = (int)(r % Wo), oy = (int)((r / Wo) % Ho), b = (int)(r / ((long long)Wo * Ho));
    float m = -INFINITY;
    for (int ky = 0; ky < 3; ++ky) {
      const int iy = 2 * oy - 1 + ky;
      if (iy < 0 || iy >= H) continue;
      for (int kx = 0; kx < 3; ++kx) {
        const int ix = 2 * ox - 1 + kx;
        if (ix < 0 || ix >= W) continue;
        const float v = __ldg(in + ((long long)(b * H + iy) * W + ix) * ldi + c);
        m = (v > m || v != v) ? v : m;      // NaN propagates, as in F.max_pool2d
      }
    }
    out[r * ldo + c] = m;
  }
}

// Positions per CTA of the position embedding: grid (B, ceil(h*w / POS_PIX)).  Every CTA resamples the whole (small) mask of
// its image, which the cumsums need, and computes and writes its own POS_PIX positions x 2 npf channels.
constexpr int POS_PIX = 32;

// Shared memory: y_embed / x_embed of the CTA's positions (normalised), dim_t [npf], not_mask [h*w] bytes.
__global__ void __launch_bounds__(256) position_sine_kernel(const uint8_t* __restrict__ mask, int Hi, int Wi, int h, int w, int npf,
                                                            float temperature, float* __restrict__ pos, int ldpos,
                                                            uint8_t* __restrict__ mask_out) {
  extern __shared__ float sh[];
  float* ye = sh;
  float* xe = sh + POS_PIX;
  float* dim_t = sh + 2 * POS_PIX;
  uint8_t* nm = reinterpret_cast<uint8_t*>(dim_t + npf);
  const int b = blockIdx.x, n = h * w, p0 = blockIdx.y * POS_PIX, np_ = min(POS_PIX, n - p0);
  // F.interpolate(m[None].float(), size=(h, w)) nearest (backbone.py:78)
  const float sy = (float)Hi / (float)h, sx = (float)Wi / (float)w;
  for (int p = threadIdx.x; p < n; p += blockDim.x) {
    const int y = p / w, x = p - y * w;
    uint8_t m = 0;
    if (mask) {
      const int iy = nearest_src(y, sy, Hi), ix = nearest_src(x, sx, Wi);
      m = mask[((long long)b * Hi + iy) * Wi + ix] != 0;
    }
    if (mask_out && p >= p0 && p < p0 + np_) mask_out[(long long)b * n + p] = m;
    nm[p] = !m;                            // not_mask, position_encoding.py:32
  }
  for (int i = threadIdx.x; i < npf; i += blockDim.x)   // temperature ** (2 * (i // 2) / npf), :41-42
    dim_t[i] = powf(temperature, (float)(2 * (i / 2)) / (float)npf);
  __syncthreads();
  // cumsum over y and x (:33-34), then / (last + 1e-6) * 2 pi (:35-38); the counts are small integers, exact in fp32
  const float scale = 6.283185307179586f, eps = 1e-6f;
  for (int q = threadIdx.x; q < np_; q += blockDim.x) {
    const int p = p0 + q, y = p / w, x = p - y * w;
    int sy_ = 0, ly = 0, sx_ = 0, lx = 0;
    for (int t = 0; t < h; ++t) { const int v = nm[t * w + x]; ly += v; if (t <= y) sy_ += v; }
    for (int t = 0; t < w; ++t) { const int v = nm[y * w + t]; lx += v; if (t <= x) sx_ += v; }
    ye[q] = (float)sy_ / ((float)ly + eps) * scale;
    xe[q] = (float)sx_ / ((float)lx + eps) * scale;
  }
  __syncthreads();
  // pos[..., j]: j < npf from y_embed, j >= npf from x_embed; even channel sin, odd channel cos (:44-47)
  const int d = 2 * npf;
  for (int i = threadIdx.x; i < np_ * d; i += blockDim.x) {
    const int q = i / d, j = i - q * d, jj = j < npf ? j : j - npf;
    const float t = (j < npf ? ye[q] : xe[q]) / dim_t[jj];
    pos[((long long)b * n + p0 + q) * ldpos + j] = (jj & 1) ? cosf(t) : sinf(t);
  }
}

int grid_for(long long total) {
  const long long cap = (long long)sm_count() * 8, g = (total + 255) / 256;
  return (int)(g < 1 ? 1 : (g < cap ? g : cap));
}

}  // namespace
}  // namespace mmx

using namespace mmx;
extern "C" {

int mmx_conv2d_dilated(const float* x, long long sN, long long sY, long long sX, long long sC, int B, int H, int W, int C,
                       const float* Wr, int ldw, const void* packed, const float* bias, const float* residual, int ldres, float* out,
                       int ldo, int Cout, int kh, int kw, int stride, int pad, int dilation, int act, void* stream) {
  MMX_REQUIRE(x && Wr && out && B > 0 && H > 0 && W > 0 && C > 0 && Cout > 0 && kh > 0 && kw > 0 && stride > 0 && pad >= 0 &&
              dilation > 0, "bad arguments");
  const int Ho = (H + 2 * pad - dilation * (kh - 1) - 1) / stride + 1, Wo = (W + 2 * pad - dilation * (kw - 1) - 1) / stride + 1;
  MMX_REQUIRE(Ho > 0 && Wo > 0, "kernel larger than the padded input");
  const long long Ml = (long long)B * Ho * Wo;
  MMX_REQUIRE(Ml < (1ll << 31) && (long long)kh * kw * C < (1 << 30), "problem too large");
  const int M = (int)Ml, K = kh * kw * C;
  MMX_REQUIRE(ldw >= K && ldo >= Cout && (!residual || ldres >= Cout), "row strides too small");
  cudaStream_t st = (cudaStream_t)stream;
  GemmEpilogue ep;
  ep.bias = bias; ep.residual = residual; ep.ldres = ldres;
  if (act != MMX_ACT_NONE) { ep.act = act; ep.C_act = out; }     // store act(C) only
  const BOperand Bop = packed_operand(Wr, ldw, packed, Cout, K);
  // 1x1, stride 1, rows of unit channel stride: the activation itself is the GEMM operand
  if (kh == 1 && kw == 1 && stride == 1 && pad == 0 && sC == 1 && sY == (long long)W * sX && sN == (long long)H * sY &&
      sX < (1 << 30))
    return gemm_nt_b(x, (int)sX, Bop, out, ldo, M, Cout, K, ep, st);
  keep_stream_scratch_cached();
  ConvGeom g{sN, sY, sX, sC, H, W, C, Ho, Wo, kw, stride, pad, dilation, M, K};
  const bool vec = C % 4 == 0 && sC == 1 && sN % 4 == 0 && sY % 4 == 0 && sX % 4 == 0 && aligned16(x);
  const long long total = (long long)M * ((K + 3) / 4);
  auto gather = [&](int ld, float* f32, __half* hi, __half* lo) {
    if (vec) im2col_kernel<true><<<grid_for(total), 256, 0, st>>>(x, g, ld, f32, hi, lo);
    else im2col_kernel<false><<<grid_for(total), 256, 0, st>>>(x, g, ld, f32, hi, lo);
  };
  if (gemm_backend() == 3 && gemm_f16x3_planes_ok(round_up(K, 8), Bop, out, ldo, Cout, K, ep)) {
    const int ldpa = round_up(K, 8);
    __half* planes = nullptr;
    MMX_CHECK_CUDA(cudaMallocAsync((void**)&planes, (size_t)2 * M * ldpa * sizeof(__half), st));
    __half *hi = planes, *lo = planes + (size_t)M * ldpa;
    gather(ldpa, nullptr, hi, lo);
    MMX_LAUNCH_CHECK();
    const int rc = gemm_nt_planes(reinterpret_cast<const uint16_t*>(hi), reinterpret_cast<const uint16_t*>(lo), ldpa, Bop, out,
                                  ldo, M, Cout, K, ep, st);
    cudaFreeAsync(planes, st);
    return rc;
  }
  // backends 0-2 (and shapes the fp16x3 kernel does not take): fp32 patches through the ordinary dispatch
  const int lda = round_up(K, 4);
  float* patches = nullptr;
  MMX_CHECK_CUDA(cudaMallocAsync((void**)&patches, (size_t)M * lda * sizeof(float), st));
  gather(lda, patches, nullptr, nullptr);
  MMX_LAUNCH_CHECK();
  const int rc = gemm_nt_b(patches, lda, Bop, out, ldo, M, Cout, K, ep, st);
  cudaFreeAsync(patches, st);
  return rc;
}

int mmx_conv2d(const float* x, long long sN, long long sY, long long sX, long long sC, int B, int H, int W, int C,
               const float* Wr, int ldw, const void* packed, const float* bias, const float* residual, int ldres, float* out,
               int ldo, int Cout, int kh, int kw, int stride, int pad, int act, void* stream) {
  return mmx_conv2d_dilated(x, sN, sY, sX, sC, B, H, W, C, Wr, ldw, packed, bias, residual, ldres, out, ldo, Cout, kh, kw, stride,
                            pad, 1, act, stream);
}

int mmx_maxpool2d_nhwc(const float* in, int ldi, float* out, int ldo, int B, int H, int W, int C, void* stream) {
  MMX_REQUIRE(in && out && B > 0 && H > 0 && W > 0 && C > 0 && ldi >= C && ldo >= C, "bad arguments");
  const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
  maxpool3s2_kernel<<<grid_for((long long)B * Ho * Wo * C), 256, 0, (cudaStream_t)stream>>>(in, ldi, out, ldo, B, H, W, C, Ho, Wo);
  MMX_LAUNCH_CHECK();
  return 0;
}

int mmx_detr_position_sine(const uint8_t* mask, int B, int Hi, int Wi, int h, int w, int npf, float temperature, float* pos,
                           int ldpos, uint8_t* mask_out, void* stream) {
  MMX_REQUIRE(pos && B > 0 && h > 0 && w > 0 && npf > 0 && ldpos >= 2 * npf, "bad arguments");
  MMX_REQUIRE(h * w <= 16384 && npf <= 2048, "feature map larger than 16384 positions");
  MMX_REQUIRE(!mask || (Hi > 0 && Wi > 0), "mask dims");
  const size_t smem = (size_t)(2 * POS_PIX + npf) * sizeof(float) + (size_t)h * w;
  const dim3 grid(B, cdiv(h * w, POS_PIX));
  position_sine_kernel<<<grid, 256, smem, (cudaStream_t)stream>>>(mask, Hi, Wi, h, w, npf, temperature, pos, ldpos, mask_out);
  MMX_LAUNCH_CHECK();
  return 0;
}
}
