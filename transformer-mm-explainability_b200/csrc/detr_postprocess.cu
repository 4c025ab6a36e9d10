// DETR's evaluation post-processors on the device (DETR/engine.py:188-192): PostProcess (DETR/models/detr.py:278-306) and
// PostProcessSegm (DETR/models/segmentation.py:218-242), plus the keep rule of the segmentation driver
// (DETR/mask_generator.py:50-51).
//
// mmx_detr_postprocess: one warp per (image, query) row of pred_logits.  The softmax follows torch's warp softmax for rows
// of up to 1024 columns (per-lane sums over columns lane, lane + 32, ..., then a butterfly), so scores are the same bits in
// practice and within 2 ulp by construction; score / label are torch's max(-1) over prob[:C] (NaN wins, ties take the lower
// index); the boxes are cxcywh -> xyxy times (w, h, w, h) with explicitly rounded operations (0.5 w is exact).
//
// mmx_detr_segm_postprocess: F.interpolate(bilinear, align_corners=False) to the batch's max size, sigmoid() > threshold,
// the crop [:img_h, :img_w] and F.interpolate(nearest) to the original size, fused into one launch.  Only the bilinear
// values the nearest step picks are computed; each query's small h x w plane is staged in shared memory and the per-column
// nearest + bilinear indices are computed once per CTA.
#include "mmx_common.cuh"

namespace mmx {
namespace {

constexpr int PP_WARPS = 8;            // rows of pred_logits per CTA of the post-process kernel
constexpr int SEGM_ROWS = 16;          // output rows per CTA of the segmentation kernel
constexpr int SEGM_MAX_IMAGES = 64;    // images per call (the per-image geometry is a kernel parameter)

__global__ void __launch_bounds__(PP_WARPS * 32) detr_postprocess_kernel(
    const float* __restrict__ logits, int ld, int rows, int Q, int C1, float keep_thr, float* __restrict__ scores,
    long long* __restrict__ labels, uint8_t* __restrict__ keep, const float* __restrict__ boxes,
    const long long* __restrict__ sizes, float* __restrict__ boxes_out) {
  const int lane = threadIdx.x & 31, r = blockIdx.x * PP_WARPS + (threadIdx.x >> 5);
  if (r >= rows) return;
  const float* x = logits + (long long)r * ld;
  // softmax over the C + 1 columns, as torch's warp softmax orders it
  float m, s;
  warp_softmax_stats(x, C1, lane, m, s);
  // max / argmax of prob[:C]; a NaN or inf logit makes every prob NaN (the sum is NaN), as in torch
  float best = 0.f;
  int bi = -1;
  for (int c = lane; c < C1 - 1; c += 32) {
    const float p = expf(x[c] - m) / s;
    if (argmax_better(p, c, best, bi)) { best = p; bi = c; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (argmax_better(ob, oi, best, bi)) { best = ob; bi = oi; }
  }
  if (lane == 0) {
    if (scores) scores[r] = best;
    if (labels) labels[r] = bi;
    if (keep) keep[r] = best > keep_thr;            // false for NaN
  }
  if (boxes_out && lane < 4) {
    // box_cxcywh_to_xyxy (DETR/util/box_ops.py:9-12) times scale_fct = (img_w, img_h, img_w, img_h) (detr.py:298-302)
    const float* bx = boxes + (long long)r * 4;
    const int yx = lane & 1;                                           // 0: x / w, 1: y / h
    const float c = bx[yx], half = __fmul_rn(0.5f, bx[2 + yx]);
    const float v = lane < 2 ? __fsub_rn(c, half) : __fadd_rn(c, half);
    const long long* sz = sizes + (long long)(r / Q) * 2;              // (img_h, img_w)
    boxes_out[(long long)r * 4 + lane] = __fmul_rn(v, (float)sz[yx ? 0 : 1]);
  }
}

struct SegmImage {
  long long offset;     // byte offset of the image's [Q, oh, ow] masks in the output
  int img_h, img_w;     // the unpadded input size (target_sizes row): the crop of the max_h x max_w bilinear grid
  int oh, ow;           // the original size (orig_target_sizes row)
};
struct SegmBatch {
  SegmImage im[SEGM_MAX_IMAGES];
};

// Grid (ceil(max oh / SEGM_ROWS), Q, B).  Shared memory: the [h, w] plane, then per output column the packed taps
// (x0 | x1 << 16) and the weight of x1, then the same per output row of the CTA.
__global__ void __launch_bounds__(256) detr_segm_kernel(const float* __restrict__ masks, int Q, int h, int w, int max_h,
                                                        int max_w, float threshold, SegmBatch batch, uint8_t* __restrict__ out) {
  extern __shared__ float sh[];
  const SegmImage im = batch.im[blockIdx.z];
  const int q = blockIdx.y, y0 = blockIdx.x * SEGM_ROWS;
  if (y0 >= im.oh) return;
  const int nrows = min(SEGM_ROWS, im.oh - y0), ow = im.ow, n = h * w;
  float* P = sh;
  int* ctap = reinterpret_cast<int*>(P + n);
  float* cl1 = reinterpret_cast<float*>(ctap + ow);
  int* rtap = reinterpret_cast<int*>(cl1 + ow);
  float* rl1 = reinterpret_cast<float*>(rtap + SEGM_ROWS);
  // F.interpolate(bilinear) of a plane to its own size is a copy in ATen (no 0 * inf terms)
  const bool copy = h == max_h && w == max_w;
  const float* src = masks + ((long long)blockIdx.z * Q + q) * n;
  for (int i = threadIdx.x; i < n; i += blockDim.x) P[i] = __ldg(src + i);
  const float sx = (float)im.img_w / (float)ow, sy = (float)im.img_h / (float)im.oh;
  const float bw = (float)w / (float)max_w, bh = (float)h / (float)max_h;
  for (int x = threadIdx.x; x < ow; x += blockDim.x) {
    const int xc = nearest_src(x, sx, im.img_w);
    int a = xc, b = xc;
    float l1 = 0.f;
    if (!copy) linear_taps(xc, bw, w, a, b, l1);
    ctap[x] = a | (b << 16);
    cl1[x] = l1;
  }
  for (int r = threadIdx.x; r < nrows; r += blockDim.x) {
    const int yc = nearest_src(y0 + r, sy, im.img_h);
    int a = yc, b = yc;
    float l1 = 0.f;
    if (!copy) linear_taps(yc, bh, h, a, b, l1);
    rtap[r] = a | (b << 16);
    rl1[r] = l1;
  }
  __syncthreads();
  // 16-byte chunks aligned in the output: a chunk wholly inside a row is one 16-byte store, the partial chunks at the two
  // ends of a row are byte stores
  uint8_t* plane = out + im.offset + (long long)q * im.oh * ow;
  const int nch = (ow + 30) / 16;                       // chunks a row of ow bytes can touch
  for (int i = threadIdx.x; i < nrows * nch; i += blockDim.x) {
    const int r = i / nch, c = i - r * nch;
    uint8_t* row = plane + (long long)(y0 + r) * ow;
    const int lead = (int)(reinterpret_cast<uintptr_t>(row) & 15);
    const int xs = c * 16 - lead;                         // first column of the chunk (may be negative)
    if (xs >= ow) continue;
    const int ry = rtap[r], ry0 = (ry & 0xffff) * w, ry1 = (ry >> 16) * w;
    const float lh1 = rl1[r], lh0 = 1.f - lh1;
    uint32_t word[4] = {0u, 0u, 0u, 0u};
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int x = xs + j;
      if (x < 0 || x >= ow) continue;
      const int cx = ctap[x], x0 = cx & 0xffff, x1 = cx >> 16;
      float v;
      if (copy) {
        v = P[ry0 + x0];
      } else {
        const float lw1 = cl1[x], lw0 = 1.f - lw1;
        v = lh0 * (lw0 * P[ry0 + x0] + lw1 * P[ry0 + x1]) + lh1 * (lw0 * P[ry1 + x0] + lw1 * P[ry1 + x1]);
      }
      const uint32_t bit = (1.f / (1.f + expf(-v))) > threshold ? 1u : 0u;   // sigmoid() > threshold, then .byte()
      word[j >> 2] |= bit << (8 * (j & 3));
    }
    if (xs >= 0 && xs + 16 <= ow) {
      *reinterpret_cast<uint4*>(row + xs) = make_uint4(word[0], word[1], word[2], word[3]);
    } else {
      for (int j = 0; j < 16; ++j) {
        const int x = xs + j;
        if (x >= 0 && x < ow) row[x] = (uint8_t)(word[j >> 2] >> (8 * (j & 3)));
      }
    }
  }
}

}  // namespace
}  // namespace mmx

using namespace mmx;
extern "C" {

int mmx_detr_postprocess(const float* logits, int ld, int B, int Q, int C1, float keep_threshold, float* scores, int64_t* labels,
                         uint8_t* keep, const float* boxes, const int64_t* sizes, float* boxes_out, void* stream) {
  MMX_REQUIRE(logits && B > 0 && Q > 0 && ld >= C1, "bad arguments");
  MMX_REQUIRE(C1 >= 2, "pred_logits needs at least one class and the no-object column (C + 1 >= 2)");
  MMX_REQUIRE(!boxes_out || (boxes && sizes), "boxes_out needs pred_boxes and the target sizes");
  MMX_REQUIRE((long long)B * Q < (1ll << 31), "too many rows");
  const int rows = B * Q;
  detr_postprocess_kernel<<<cdiv(rows, PP_WARPS), PP_WARPS * 32, 0, (cudaStream_t)stream>>>(
      logits, ld, rows, Q, C1, keep_threshold, scores, reinterpret_cast<long long*>(labels), keep, boxes,
      reinterpret_cast<const long long*>(sizes), boxes_out);
  MMX_LAUNCH_CHECK();
  return 0;
}

int mmx_detr_segm_postprocess(const float* pred_masks, int B, int Q, int h, int w, const int* sizes, const int* orig_sizes,
                              float threshold, uint8_t* out, void* stream) {
  MMX_REQUIRE(pred_masks && out && sizes && orig_sizes && B > 0 && Q > 0 && w > 0, "bad arguments");
  MMX_REQUIRE(h > 1, "pred_masks [B, Q, h, w] needs h > 1 (the reference's squeeze(2) drops a height of 1)");
  MMX_REQUIRE(h < 65536 && w < 65536 && Q < 65536, "mask plane or query count too large");
  MMX_REQUIRE(B <= SEGM_MAX_IMAGES, "at most 64 images per call");
  SegmBatch batch;
  int max_h = 0, max_w = 0, max_oh = 0, max_ow = 0;
  long long offset = 0;
  for (int i = 0; i < B; ++i) {
    const int ih = sizes[2 * i], iw = sizes[2 * i + 1], oh = orig_sizes[2 * i], ow = orig_sizes[2 * i + 1];
    MMX_REQUIRE(ih > 0 && iw > 0 && oh > 0 && ow > 0, "image sizes must be positive");
    batch.im[i] = SegmImage{offset, ih, iw, oh, ow};
    offset += (long long)Q * oh * ow;
    // (max_h, max_w) is the column max of the sizes, so every image's crop lies inside the bilinear grid
    max_h = max(max_h, ih); max_w = max(max_w, iw); max_oh = max(max_oh, oh); max_ow = max(max_ow, ow);
  }
  const size_t smem = (size_t)h * w * sizeof(float) + (size_t)max_ow * 8 + (size_t)SEGM_ROWS * 8;
  MMX_REQUIRE(smem <= 200 * 1024, "mask plane plus the per-column taps exceed shared memory");
  if (smem > 48 * 1024)
    MMX_CHECK_CUDA(cudaFuncSetAttribute(detr_segm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const dim3 grid(cdiv(max_oh, SEGM_ROWS), Q, B);
  detr_segm_kernel<<<grid, 256, smem, (cudaStream_t)stream>>>(pred_masks, Q, h, w, max_h, max_w, threshold, batch, out);
  MMX_LAUNCH_CHECK();
  return 0;
}
}
