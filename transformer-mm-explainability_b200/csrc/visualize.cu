// The notebooks' last step, on the device: turning a relevance map into the picture a person looks at.
//   relevance overlay   CLIP_explainability.ipynb show_image_relevance, Transformer_MM_explainability_ViT.ipynb
//                       generate_visualization: bilinear upsample, min-max, cv2 JET heat map + image, / max, uint8, RGB<->BGR
//   box relevance image LXMERT.ipynb save_image_vis: per-box max into a full-resolution mask, min-max, * image, imwrite's 8U
//   CLIP text scores    CLIP_explainability.ipynb show_heatmap_on_text: R_text[eot, 1:eot] / R_text[eot, 1:eot].sum()
//
// The two image kernels need whole-picture reductions (min / max) between elementwise passes.  One thread-block cluster
// of VIS_CLUSTER CTAs owns one picture: each CTA reduces its share, the partials are exchanged through distributed shared
// memory (every CTA reads all of them, in rank order), so a picture is one launch whatever the batch size, with no global
// scratch, no atomics and no host synchronisation.  Every pass recomputes its per-pixel values from the inputs (the map
// grid, the boxes and the JET table sit in shared memory; the image is re-read, from L2) instead of staging the picture.
// All arithmetic is fp32 with explicitly rounded operations, in the reference's order.
#include <cooperative_groups.h>

#include "mmx_common.cuh"

namespace cg = cooperative_groups;

namespace mmx {
namespace {

constexpr int VIS_CLUSTER = 8;
constexpr int VIS_THREADS = 256;
constexpr int VIS_MAX_GRID = 64 * 64;   // the h x w map staged in shared memory
constexpr int VIS_MAX_BOXES = 1024;

// cv2.applyColorMap(x, COLORMAP_JET) for x = 0 .. 255, BGR (OpenCV's colormap.cpp interpolates its JET control points to
// these 256 entries; the table is pinned by a golden of cv2's own output).
__constant__ unsigned char c_jet[256 * 3] = {
128, 0, 0, 132, 0, 0, 136, 0, 0, 140, 0, 0, 144, 0, 0, 148, 0, 0, 152, 0, 0, 156, 0, 0, 160, 0, 0, 164, 0, 0, 168, 0,
0, 172, 0, 0, 176, 0, 0, 180, 0, 0, 184, 0, 0, 188, 0, 0, 192, 0, 0, 196, 0, 0, 200, 0, 0, 204, 0, 0, 208, 0, 0, 212,
0, 0, 216, 0, 0, 220, 0, 0, 224, 0, 0, 228, 0, 0, 232, 0, 0, 236, 0, 0, 240, 0, 0, 244, 0, 0, 248, 0, 0, 252, 0, 0,
255, 0, 0, 255, 4, 0, 255, 8, 0, 255, 12, 0, 255, 16, 0, 255, 20, 0, 255, 24, 0, 255, 28, 0, 255, 32, 0, 255, 36, 0,
255, 40, 0, 255, 44, 0, 255, 48, 0, 255, 52, 0, 255, 56, 0, 255, 60, 0, 255, 64, 0, 255, 68, 0, 255, 72, 0, 255, 76,
0, 255, 80, 0, 255, 84, 0, 255, 88, 0, 255, 92, 0, 255, 96, 0, 255, 100, 0, 255, 104, 0, 255, 108, 0, 255, 112, 0,
255, 116, 0, 255, 120, 0, 255, 124, 0, 255, 128, 0, 255, 132, 0, 255, 136, 0, 255, 140, 0, 255, 144, 0, 255, 148, 0,
255, 152, 0, 255, 156, 0, 255, 160, 0, 255, 164, 0, 255, 168, 0, 255, 172, 0, 255, 176, 0, 255, 180, 0, 255, 184, 0,
255, 188, 0, 255, 192, 0, 255, 196, 0, 255, 200, 0, 255, 204, 0, 255, 208, 0, 255, 212, 0, 255, 216, 0, 255, 220, 0,
255, 224, 0, 255, 228, 0, 255, 232, 0, 255, 236, 0, 255, 240, 0, 255, 244, 0, 255, 248, 0, 255, 252, 0, 254, 255, 2,
250, 255, 6, 246, 255, 10, 242, 255, 14, 238, 255, 18, 234, 255, 22, 230, 255, 26, 226, 255, 30, 222, 255, 34, 218,
255, 38, 214, 255, 42, 210, 255, 46, 206, 255, 50, 202, 255, 54, 198, 255, 58, 194, 255, 62, 190, 255, 66, 186, 255,
70, 182, 255, 74, 178, 255, 78, 174, 255, 82, 170, 255, 86, 166, 255, 90, 162, 255, 94, 158, 255, 98, 154, 255, 102,
150, 255, 106, 146, 255, 110, 142, 255, 114, 138, 255, 118, 134, 255, 122, 130, 255, 126, 126, 255, 130, 122, 255,
134, 118, 255, 138, 114, 255, 142, 110, 255, 146, 106, 255, 150, 102, 255, 154, 98, 255, 158, 94, 255, 162, 90, 255,
166, 86, 255, 170, 82, 255, 174, 78, 255, 178, 74, 255, 182, 70, 255, 186, 66, 255, 190, 62, 255, 194, 58, 255, 198,
54, 255, 202, 50, 255, 206, 46, 255, 210, 42, 255, 214, 38, 255, 218, 34, 255, 222, 30, 255, 226, 26, 255, 230, 22,
255, 234, 18, 255, 238, 14, 255, 242, 10, 255, 246, 6, 255, 250, 1, 255, 254, 0, 252, 255, 0, 248, 255, 0, 244, 255,
0, 240, 255, 0, 236, 255, 0, 232, 255, 0, 228, 255, 0, 224, 255, 0, 220, 255, 0, 216, 255, 0, 212, 255, 0, 208, 255,
0, 204, 255, 0, 200, 255, 0, 196, 255, 0, 192, 255, 0, 188, 255, 0, 184, 255, 0, 180, 255, 0, 176, 255, 0, 172, 255,
0, 168, 255, 0, 164, 255, 0, 160, 255, 0, 156, 255, 0, 152, 255, 0, 148, 255, 0, 144, 255, 0, 140, 255, 0, 136, 255,
0, 132, 255, 0, 128, 255, 0, 124, 255, 0, 120, 255, 0, 116, 255, 0, 112, 255, 0, 108, 255, 0, 104, 255, 0, 100, 255,
0, 96, 255, 0, 92, 255, 0, 88, 255, 0, 84, 255, 0, 80, 255, 0, 76, 255, 0, 72, 255, 0, 68, 255, 0, 64, 255, 0, 60,
255, 0, 56, 255, 0, 52, 255, 0, 48, 255, 0, 44, 255, 0, 40, 255, 0, 36, 255, 0, 32, 255, 0, 28, 255, 0, 24, 255, 0,
20, 255, 0, 16, 255, 0, 12, 255, 0, 8, 255, 0, 4, 255, 0, 0, 255, 0, 0, 252, 0, 0, 248, 0, 0, 244, 0, 0, 240, 0, 0,
236, 0, 0, 232, 0, 0, 228, 0, 0, 224, 0, 0, 220, 0, 0, 216, 0, 0, 212, 0, 0, 208, 0, 0, 204, 0, 0, 200, 0, 0, 196, 0,
0, 192, 0, 0, 188, 0, 0, 184, 0, 0, 180, 0, 0, 176, 0, 0, 172, 0, 0, 168, 0, 0, 164, 0, 0, 160, 0, 0, 156, 0, 0, 152,
0, 0, 148, 0, 0, 144, 0, 0, 140, 0, 0, 136, 0, 0, 132, 0, 0, 128};

// Min and max (NaN-propagating, as np.min / np.max and torch's min() / max()) of the whole picture: the CTA's partials
// are reduced in the CTA, published in slot `slot` of every CTA's `part`, and after the cluster barrier each CTA reads the
// VIS_CLUSTER partials in rank order.  Every thread gets both results.  `part` holds two slots per CTA, so the second
// reduction of a kernel never overwrites a partial another CTA may still be reading from the first.
__device__ __forceinline__ void cluster_minmax_nan(float& mn, float& mx, float2* part, int slot) {
  __shared__ float2 warp_part[VIS_THREADS / 32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    mn = min_nan(mn, __shfl_xor_sync(0xffffffffu, mn, o));
    mx = max_nan(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  }
  if ((threadIdx.x & 31) == 0) warp_part[threadIdx.x >> 5] = make_float2(mn, mx);
  __syncthreads();
  if (threadIdx.x == 0) {
    float a = warp_part[0].x, b = warp_part[0].y;
#pragma unroll
    for (int w = 1; w < VIS_THREADS / 32; ++w) { a = min_nan(a, warp_part[w].x); b = max_nan(b, warp_part[w].y); }
    part[slot] = make_float2(a, b);
  }
  cg::cluster_group cluster = cg::this_cluster();
  cluster.sync();
  mn = INFINITY; mx = -INFINITY;
#pragma unroll
  for (int r = 0; r < VIS_CLUSTER; ++r) {
    const float2 p = cluster.map_shared_rank(part, r)[slot];
    mn = min_nan(mn, p.x); mx = max_nan(mx, p.y);
  }
}

// (v - mn) / d then * 255, as the numpy expressions compute it, cast to uint8 with numpy's truncation (NaN -> 0, as the
// cast gives on x86; the value never exceeds 255 because (v - mn) <= d).
__device__ __forceinline__ int quant255(float v) { return v >= 0.f ? (int)v & 255 : 0; }

// [lo, hi) of the range a CTA of the cluster owns when n items are split into VIS_CLUSTER near-equal parts
__device__ __forceinline__ void cta_range(long long n, int rank, long long& lo, long long& hi) {
  lo = n * rank / VIS_CLUSTER;
  hi = n * (rank + 1) / VIS_CLUSTER;
}

struct OverlayPixel {
  const float* grid;     // [h, w]: in shared memory, or the map in global memory when it is copied (h, w = H, W)
  const float* heat;     // [256, 3] JET / 255 in shared memory
  const float* img;      // [3, H, W] of this picture's image
  int h, w, W;
  long long HW;
  float sh, sw;
  bool copy;

  // F.interpolate(mode="bilinear", align_corners=False) at output pixel p: upsample_bilinear2d_out_frame's expression
  // (ATen, UpSampleBilinear2d.cu) h0 (w0 a + w1 b) + h1 (w0 c + w1 d) with the contraction torch's CUDA build applies,
  // written out: each sum is an fma on its first product (of the eight ways to contract it, the only one that matched
  // torch 2.11's F.interpolate bit for bit on an H100).  A copy when the sizes match.
  __device__ __forceinline__ float up(long long p) const {
    const int y = (int)(p / W), x = (int)(p - (long long)y * W);
    if (copy) return __ldg(grid + p);
    int y0, y1, x0, x1;
    float ly1, lx1;
    linear_taps(y, sh, h, y0, y1, ly1);
    linear_taps(x, sw, w, x0, x1, lx1);
    const float ly0 = 1.f - ly1, lx0 = 1.f - lx1;
    const float* r0 = grid + y0 * w;
    const float* r1 = grid + y1 * w;
    const float t0 = __fmaf_rn(lx0, r0[x0], __fmul_rn(lx1, r0[x1]));
    const float t1 = __fmaf_rn(lx0, r1[x0], __fmul_rn(lx1, r1[x1]));
    return __fmaf_rn(ly0, t0, __fmul_rn(ly1, t1));
  }
  // show_cam_on_image's cam = heatmap / 255 + img at pixel p, channel c: the heat map's BGR channel c meets the image's RGB
  // channel c, as in the reference
  __device__ __forceinline__ void cam(long long p, float mn, float d, float imn, float id, float out[3]) const {
    const int q = quant255(__fmul_rn(__fdiv_rn(__fsub_rn(up(p), mn), d), 255.f));
#pragma unroll
    for (int c = 0; c < 3; ++c)
      out[c] = __fadd_rn(heat[q * 3 + c], __fdiv_rn(__fsub_rn(__ldg(img + c * HW + p), imn), id));
  }
};

// One cluster per map b.  Pass 1: min / max of the upsampled map and of the image (three channels).  Pass 2: max of the
// cam.  Pass 3: uint8(255 * cam / max) with the channels reversed, written in 16-byte chunks of the [H, W, 3] picture.
__global__ void __cluster_dims__(VIS_CLUSTER, 1, 1) __launch_bounds__(VIS_THREADS)
relevance_overlay_kernel(const float* __restrict__ rel, int h, int w, float sh, float sw, const float* __restrict__ images,
                         int n_img, int H, int W, unsigned char* __restrict__ out) {
  __shared__ float s_grid[VIS_MAX_GRID];
  __shared__ float s_heat[256 * 3];
  __shared__ float2 s_part[2];
  const int rank = (int)cg::this_cluster().block_rank();
  const int b = blockIdx.x / VIS_CLUSTER;
  const long long HW = (long long)H * W;
  const int n = (int)min((long long)h * w, (long long)VIS_MAX_GRID);
  const bool copy = h == H && w == W;
  const float* map = rel + (long long)b * h * w;
  if (!copy)
    for (int i = threadIdx.x; i < n; i += VIS_THREADS) s_grid[i] = __ldg(map + i);
  for (int i = threadIdx.x; i < 256 * 3; i += VIS_THREADS) s_heat[i] = __fdiv_rn((float)c_jet[i], 255.f);
  __syncthreads();
  OverlayPixel px{copy ? map : s_grid, s_heat, images + (n_img == 1 ? 0 : (long long)b * 3 * HW), h, w, W, HW, sh, sw,
                  copy};

  long long p0, p1;
  cta_range(HW, rank, p0, p1);
  float mn = INFINITY, mx = -INFINITY, imn = INFINITY, imx = -INFINITY;
  for (long long p = p0 + threadIdx.x; p < p1; p += VIS_THREADS) {
    const float v = px.up(p);
    mn = min_nan(mn, v); mx = max_nan(mx, v);
#pragma unroll
    for (int c = 0; c < 3; ++c) { const float x = __ldg(px.img + c * HW + p); imn = min_nan(imn, x); imx = max_nan(imx, x); }
  }
  cluster_minmax_nan(mn, mx, s_part, 0);
  // the image's partials go through the same exchange: a second barrier, but no second pass over the pixels
  __syncthreads();
  cluster_minmax_nan(imn, imx, s_part, 1);
  const float d = __fsub_rn(mx, mn), id = __fsub_rn(imx, imn);

  float cmax = -INFINITY, unused = INFINITY;
  for (long long p = p0 + threadIdx.x; p < p1; p += VIS_THREADS) {
    float cam[3];
    px.cam(p, mn, d, imn, id, cam);
#pragma unroll
    for (int c = 0; c < 3; ++c) cmax = max_nan(cmax, cam[c]);
  }
  // slot 0 is free again: every CTA read it before the barrier of the image exchange
  __syncthreads();
  cluster_minmax_nan(unused, cmax, s_part, 0);

  // bytes of this picture, in 16-byte chunks aligned in memory; the chunks at the two ends may be partial
  unsigned char* pic = out + (long long)b * HW * 3;
  const long long nbytes = HW * 3;
  const int lead = (int)(reinterpret_cast<uintptr_t>(pic) & 15);
  const long long nch = (nbytes + lead + 15) / 16;
  long long c0, c1;
  cta_range(nch, rank, c0, c1);
  for (long long ch = c0 + threadIdx.x; ch < c1; ch += VIS_THREADS) {
    const long long k0 = ch * 16 - lead;
    uint32_t word[4] = {0u, 0u, 0u, 0u};
    long long cur = -1;
    float cam[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const long long k = k0 + j;
      if (k < 0 || k >= nbytes) continue;
      const long long p = k / 3;
      if (p != cur) { px.cam(p, mn, d, imn, id, cam); cur = p; }
      const int c = (int)(k - p * 3);                       // output channel c holds vis channel 2 - c (cvtColor RGB2BGR)
      const float cv = c == 0 ? cam[2] : c == 1 ? cam[1] : cam[0];
      const uint32_t v = (uint32_t)quant255(__fmul_rn(255.f, __fdiv_rn(cv, cmax)));
      word[j >> 2] |= v << (8 * (j & 3));
    }
    if (k0 >= 0 && k0 + 16 <= nbytes) {
      *reinterpret_cast<uint4*>(pic + k0) = make_uint4(word[0], word[1], word[2], word[3]);
    } else {
      for (int j = 0; j < 16; ++j) {
        const long long k = k0 + j;
        if (k >= 0 && k < nbytes) pic[k] = (unsigned char)(word[j >> 2] >> (8 * (j & 3)));
      }
    }
  }
  cg::this_cluster().sync();   // no CTA leaves while another may still read its partials
}

// Python / torch slice bound of int(v) (truncation toward zero) on an axis of n: a negative bound wraps once, then the
// bound clamps to [0, n].  Coordinates beyond +-2^30 are clamped first so the conversion cannot overflow.
__device__ __forceinline__ int slice_bound(float v, int n) {
  const float t = fminf(fmaxf(truncf(v), -1073741824.f), 1073741824.f);
  int i = (int)t;
  if (i < 0) { i += n; if (i < 0) i = 0; }
  return i > n ? n : i;
}

struct BoxMask {
  const int4* box;       // [n_boxes] (x0, y0, x1, y1) slice bounds in shared memory
  const float* score;
  int n_boxes, W;
  // mask[y, x] after the reference's loop: starts at 0, each covering box applies torch.max(score, mask), which
  // propagates NaN
  __device__ __forceinline__ float at(long long p) const {
    const int y = (int)(p / W), x = (int)(p - (long long)y * W);
    float m = 0.f;
    for (int i = 0; i < n_boxes; ++i) {
      const int4 bx = box[i];
      if (x >= bx.x && x < bx.z && y >= bx.y && y < bx.w) m = max_nan(m, score[i]);
    }
    return m;
  }
};

// OpenCV's float -> 8U conversion (Mat::convertTo, which imwrite applies to a float image): round half to even to int32,
// then saturate.  x86's conversion gives INT_MIN for NaN, infinities and anything beyond int32, so those give 0.
__device__ __forceinline__ uint32_t cv_saturate_u8(float v) {
  if (!(fabsf(v) < 2147483648.f)) return 0u;
  const int r = __float2int_rn(v);
  return (uint32_t)(r < 0 ? 0 : r > 255 ? 255 : r);
}

// One cluster per question b.  Pass 1: min / max of the mask.  Pass 2: img * (mask - min) / (max - min) in fp32, to 8 bits,
// in 16-byte chunks of the [H, W, 3] picture.
__global__ void __cluster_dims__(VIS_CLUSTER, 1, 1) __launch_bounds__(VIS_THREADS)
box_relevance_kernel(const unsigned char* __restrict__ img, int n_img, int H, int W, const float* __restrict__ boxes,
                     const float* __restrict__ scores, int n_boxes, unsigned char* __restrict__ out) {
  __shared__ int4 s_box[VIS_MAX_BOXES];
  __shared__ float s_score[VIS_MAX_BOXES];
  __shared__ float2 s_part[2];
  const int rank = (int)cg::this_cluster().block_rank();
  const int b = blockIdx.x / VIS_CLUSTER;
  for (int i = threadIdx.x; i < n_boxes; i += VIS_THREADS) {
    const float* bx = boxes + ((long long)b * n_boxes + i) * 4;
    s_box[i] = make_int4(slice_bound(bx[0], W), slice_bound(bx[1], H), slice_bound(bx[2], W), slice_bound(bx[3], H));
    s_score[i] = scores[(long long)b * n_boxes + i];
  }
  __syncthreads();
  const BoxMask mask{s_box, s_score, n_boxes, W};
  const long long HW = (long long)H * W;

  long long p0, p1;
  cta_range(HW, rank, p0, p1);
  float mn = INFINITY, mx = -INFINITY;
  for (long long p = p0 + threadIdx.x; p < p1; p += VIS_THREADS) {
    const float m = mask.at(p);
    mn = min_nan(mn, m); mx = max_nan(mx, m);
  }
  cluster_minmax_nan(mn, mx, s_part, 0);
  const float d = __fsub_rn(mx, mn);

  const unsigned char* src = img + (n_img == 1 ? 0 : (long long)b * HW * 3);
  unsigned char* pic = out + (long long)b * HW * 3;
  const long long nbytes = HW * 3;
  const int lead = (int)(reinterpret_cast<uintptr_t>(pic) & 15);
  const long long nch = (nbytes + lead + 15) / 16;
  long long c0, c1;
  cta_range(nch, rank, c0, c1);
  for (long long ch = c0 + threadIdx.x; ch < c1; ch += VIS_THREADS) {
    const long long k0 = ch * 16 - lead;
    uint32_t word[4] = {0u, 0u, 0u, 0u};
    long long cur = -1;
    float m = 0.f;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const long long k = k0 + j;
      if (k < 0 || k >= nbytes) continue;
      const long long p = k / 3;
      if (p != cur) { m = __fdiv_rn(__fsub_rn(mask.at(p), mn), d); cur = p; }
      word[j >> 2] |= cv_saturate_u8(__fmul_rn((float)__ldg(src + k), m)) << (8 * (j & 3));
    }
    if (k0 >= 0 && k0 + 16 <= nbytes) {
      *reinterpret_cast<uint4*>(pic + k0) = make_uint4(word[0], word[1], word[2], word[3]);
    } else {
      for (int j = 0; j < 16; ++j) {
        const long long k = k0 + j;
        if (k >= 0 && k < nbytes) pic[k] = (unsigned char)(word[j >> 2] >> (8 * (j & 3)));
      }
    }
  }
  cg::this_cluster().sync();
}

// One warp per prompt: eot = first argmax of the token row; scores[b, j] = R[b, eot, 1 + j] / s for j < eot - 1, where s is
// the slice's sum in double (lane-strided partials, then a butterfly: a fixed order) rounded once to fp32; the rest of
// the row is 0.
__global__ void __launch_bounds__(128) clip_text_scores_kernel(const float* __restrict__ R, const int* __restrict__ tokens,
                                                               int B, int ctx, float* __restrict__ scores, int* __restrict__ lens) {
  const int b = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (b >= B) return;
  const int* tok = tokens + (long long)b * ctx;
  int best = -1, bi = -1;
  for (int j = lane; j < ctx; j += 32) { const int t = tok[j]; if (bi < 0 || t > best) { best = t; bi = j; } }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const int ob = __shfl_xor_sync(0xffffffffu, best, o), oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (oi >= 0 && (bi < 0 || ob > best || (ob == best && oi < bi))) { best = ob; bi = oi; }
  }
  const int eot = bi, len = eot > 1 ? eot - 1 : 0;
  const float* row = R + ((long long)b * ctx + eot) * ctx + 1;
  double s = 0.0;
  for (int j = lane; j < len; j += 32) s += (double)row[j];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float sf = (float)s;
  float* dst = scores + (long long)b * ctx;
  for (int j = lane; j < ctx; j += 32) dst[j] = j < len ? __fdiv_rn(row[j], sf) : 0.f;
  if (lane == 0) lens[b] = len;
}

}  // namespace
}  // namespace mmx

using namespace mmx;
extern "C" {

int mmx_relevance_overlay(const float* rel, int B, int h, int w, float scale_h, float scale_w, const float* images, int n_img,
                          int H, int W, unsigned char* out, void* stream) {
  MMX_REQUIRE(rel && images && out && B > 0 && h > 0 && w > 0 && H > 0 && W > 0, "bad arguments");
  MMX_REQUIRE(n_img == 1 || n_img == B, "images must hold 1 image or B images");
  MMX_REQUIRE((long long)H * W < (1ll << 40), "picture too large");
  MMX_REQUIRE((h == H && w == W) || (long long)h * w <= VIS_MAX_GRID,
              "a map that is upsampled may hold at most 64 x 64 patches");
  MMX_REQUIRE(B <= 0x7fffffff / VIS_CLUSTER, "too many maps");
  relevance_overlay_kernel<<<B * VIS_CLUSTER, VIS_THREADS, 0, (cudaStream_t)stream>>>(rel, h, w, scale_h, scale_w, images,
                                                                                     n_img, H, W, out);
  MMX_LAUNCH_CHECK();
  return 0;
}

int mmx_box_relevance_image(const unsigned char* img, int n_img, int H, int W, const float* boxes, const float* scores, int B,
                            int n_boxes, unsigned char* out, void* stream) {
  MMX_REQUIRE(img && boxes && scores && out && B > 0 && H > 0 && W > 0 && n_boxes >= 0, "bad arguments");
  MMX_REQUIRE(n_img == 1 || n_img == B, "img must hold 1 image or B images");
  MMX_REQUIRE(n_boxes <= VIS_MAX_BOXES, "at most 1024 boxes per image");
  MMX_REQUIRE((long long)H * W < (1ll << 40), "picture too large");
  MMX_REQUIRE(B <= 0x7fffffff / VIS_CLUSTER, "too many images");
  box_relevance_kernel<<<B * VIS_CLUSTER, VIS_THREADS, 0, (cudaStream_t)stream>>>(img, n_img, H, W, boxes, scores, n_boxes, out);
  MMX_LAUNCH_CHECK();
  return 0;
}

int mmx_clip_text_scores(const float* R_text, const int* tokens, int B, int ctx, float* scores, int* lens, void* stream) {
  MMX_REQUIRE(R_text && tokens && scores && lens && B > 0 && ctx > 0, "bad arguments");
  clip_text_scores_kernel<<<cdiv(B, 4), 128, 0, (cudaStream_t)stream>>>(R_text, tokens, B, ctx, scores, lens);
  MMX_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
