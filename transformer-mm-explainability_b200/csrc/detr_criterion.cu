// DETR's evaluation losses on the device: HungarianMatcher (DETR/models/matcher.py) and SetCriterion
// (DETR/models/detr.py:103-275, DETR/models/segmentation.py:172-215) for the last decoder layer and the auxiliary ones.
//
// Layout shared by the entry points.  L layers (layer 0: the model's final output, 1 .. L-1: aux_outputs 0 .. L-2), B
// images, Q queries, C1 = num_classes + 1 logit columns.  Targets are concatenated over the images (labels [T], cxcywh
// boxes [T, 4]) with off[b] .. off[b+1] the targets of image b (host array, off[B] = T).  The cost of (layer l, image b) is
// the row-major [Q, T_b] block at l Q T + Q off[b] (the blocks the reference keeps after C.split(sizes)).  The matched
// indices of layer l are indices[l][0][off[b] + k] (query, ascending) and indices[l][1][off[b] + k] (target),
// k < min(Q, T_b); unused slots hold -1.
//
// mmx_detr_match_cost: one warp per (layer, image, query) row: the softmax (warp_softmax_stats, the order of
// mmx_detr_postprocess), then C = w_bbox cdist_L1 + w_class (-prob[tgt]) + w_giou (-GIoU) with box_ops' operation order
// and explicitly rounded operations.  status[l] gets bit 1 when a predicted box of layer l or a target box fails
// generalized_box_iou's x1 >= x0, y1 >= y0 assert (NaN included), bit 2 when a label is outside [0, C1).
//
// mmx_detr_match_lsa: one CTA per (layer, image) problem: scipy's linear_sum_assignment (rectangular_lsap, the shortest
// augmenting path of Crouse 2016) restated in double: the transpose of a tall matrix, rows taken in order, the reversed
// column scan order and the tie rule of the Dijkstra step, the dual updates and the output order.  status gets 1 for a NaN
// or -inf entry, 2 for an infeasible matrix.
//
// mmx_detr_set_losses: one CTA per layer: loss_ce (weighted NLL over the B Q rows), class_error, cardinality_error,
// loss_bbox and loss_giou; every sum is a double reduced in a fixed order.
//
// mmx_detr_mask_losses: the last layer's focal and dice losses.  One pass over the pixels of the padded target size: the
// bilinear upsample of each matched [h, w] plane (ATen's arithmetic, linear_taps), the target read in place (zero beyond
// its image), then per-(mask, row chunk) double partials reduced in a fixed order by a second launch.
#include "mmx_common.cuh"

namespace mmx {
namespace {

constexpr int CRIT_MAX_LAYERS = 16;
constexpr int CRIT_MAX_IMAGES = 64;
constexpr int LSA_MAX = 1024;          // max(Q, T_b) of one assignment problem
constexpr int LSA_THREADS = 128;
constexpr int COST_WARPS = 8;
constexpr int LOSS_THREADS = 256;
constexpr int MASK_ROWS = 8;           // target rows per CTA of the mask-loss kernel
constexpr int MASK_THREADS = 256;

struct Offsets {
  int o[CRIT_MAX_IMAGES + 1];
};
struct Layers {
  const float* logits[CRIT_MAX_LAYERS];
  const float* boxes[CRIT_MAX_LAYERS];
};

// box_cxcywh_to_xyxy (DETR/util/box_ops.py:9-13)
__device__ __forceinline__ void xyxy(const float* b, float& x0, float& y0, float& x1, float& y1) {
  const float hw = __fmul_rn(0.5f, b[2]), hh = __fmul_rn(0.5f, b[3]);
  x0 = __fsub_rn(b[0], hw); y0 = __fsub_rn(b[1], hh);
  x1 = __fadd_rn(b[0], hw); y1 = __fadd_rn(b[1], hh);
}
// generalized_box_iou's assert (box_ops.py:51-52): false for a degenerate or NaN box
__device__ __forceinline__ bool box_ok(const float* b) {
  float x0, y0, x1, y1;
  xyxy(b, x0, y0, x1, y1);
  return x1 >= x0 && y1 >= y0;
}
// torch.max / torch.min / clamp(min=0) with NaN propagation
__device__ __forceinline__ float tmax(float a, float b) { return (a != a || a > b) ? a : b; }
__device__ __forceinline__ float tmin(float a, float b) { return (a != a || a < b) ? a : b; }
__device__ __forceinline__ float clamp0(float a) { return a < 0.f ? 0.f : a; }

// generalized_box_iou of one (cxcywh) pair in box_ops' order (:22-68): areas, intersection, union, iou, enclosing area
__device__ float giou(const float* p, const float* t) {
  float a0, a1, a2, a3, b0, b1, b2, b3;
  xyxy(p, a0, a1, a2, a3);
  xyxy(t, b0, b1, b2, b3);
  const float area1 = __fmul_rn(__fsub_rn(a2, a0), __fsub_rn(a3, a1));
  const float area2 = __fmul_rn(__fsub_rn(b2, b0), __fsub_rn(b3, b1));
  const float iw = clamp0(__fsub_rn(tmin(a2, b2), tmax(a0, b0))), ih = clamp0(__fsub_rn(tmin(a3, b3), tmax(a1, b1)));
  const float inter = __fmul_rn(iw, ih);
  const float uni = __fsub_rn(__fadd_rn(area1, area2), inter);
  const float iou = __fdiv_rn(inter, uni);
  const float ew = clamp0(__fsub_rn(tmax(a2, b2), tmin(a0, b0))), eh = clamp0(__fsub_rn(tmax(a3, b3), tmin(a1, b1)));
  const float area = __fmul_rn(ew, eh);
  return __fsub_rn(iou, __fdiv_rn(__fsub_rn(area, uni), area));
}

// Grid (ceil(Q / COST_WARPS), B, L); warp = query row.
__global__ void __launch_bounds__(COST_WARPS * 32) match_cost_kernel(
    Layers lay, int B, int Q, int C1, const long long* __restrict__ tgt_ids, const float* __restrict__ tgt_boxes,
    Offsets off, float w_class, float w_bbox, float w_giou, float* __restrict__ cost, int* __restrict__ status) {
  const int l = blockIdx.z, b = blockIdx.y, lane = threadIdx.x & 31;
  const int q = blockIdx.x * COST_WARPS + (threadIdx.x >> 5);
  const int T = off.o[B], t0 = off.o[b], Tb = off.o[b + 1] - t0;
  int bad = 0;
  if (blockIdx.x == 0 && l == 0)       // the target boxes, checked once
    for (int j = threadIdx.x; j < Tb; j += blockDim.x) {
      if (!box_ok(tgt_boxes + (long long)(t0 + j) * 4)) bad |= 1;
      const long long c = tgt_ids[t0 + j];
      if (c < 0 || c >= C1) bad |= 2;
    }
  if (bad) atomicOr(status, bad);      // every layer's matcher checks the same targets: status[0] stands for all
  if (q >= Q) return;
  const long long row = (long long)b * Q + q;
  const float* x = lay.logits[l] + row * C1;
  const float* pb = lay.boxes[l] + row * 4;
  if (lane == 0 && !box_ok(pb)) atomicOr(status + l, 1);
  float m, s;
  warp_softmax_stats(x, C1, lane, m, s);
  float* out = cost + (long long)l * Q * T + (long long)Q * t0 + (long long)q * Tb;
  for (int j = lane; j < Tb; j += 32) {
    const long long c = tgt_ids[t0 + j];
    const float prob = (c >= 0 && c < C1) ? __fdiv_rn(expf(x[c] - m), s) : __int_as_float(0x7fc00000);
    const float* tb = tgt_boxes + (long long)(t0 + j) * 4;
    float l1 = 0.f;                                          // torch.cdist(p=1)
#pragma unroll
    for (int k = 0; k < 4; ++k) l1 = __fadd_rn(l1, fabsf(__fsub_rn(pb[k], tb[k])));
    const float g = giou(pb, tb);
    out[j] = __fadd_rn(__fadd_rn(__fmul_rn(w_bbox, l1), __fmul_rn(w_class, -prob)), __fmul_rn(w_giou, -g));
  }
}

// The Dijkstra step's choice among the remaining columns (rectangular_lsap.cpp augmenting_path): the lowest shortest-path
// cost; among equal ones the LAST position of an unassigned column when there is one, else the FIRST position.  This is
// the sequential scan `spc < lowest || (spc == lowest && row4col == -1)` as an associative combine.
struct Pick {
  double v;
  int it, free_;
};
__device__ __forceinline__ bool pick_better(const Pick& a, const Pick& b) {
  if (b.it < 0) return a.it >= 0;
  if (a.it < 0) return false;
  if (a.v != b.v) return a.v < b.v;
  if (a.free_ != b.free_) return a.free_ > b.free_;
  return a.free_ ? a.it > b.it : a.it < b.it;
}

__global__ void __launch_bounds__(LSA_THREADS) lsa_kernel(const float* __restrict__ cost, int B, int Q, Offsets off,
                                                          long long* __restrict__ indices, int* __restrict__ status) {
  __shared__ double u[LSA_MAX], v[LSA_MAX], spc[LSA_MAX];
  __shared__ short path[LSA_MAX], col4row[LSA_MAX], row4col[LSA_MAX], remaining[LSA_MAX];
  __shared__ bool SR[LSA_MAX], SC[LSA_MAX];
  __shared__ Pick wbest[LSA_THREADS / 32];
  __shared__ int s_index;
  __shared__ double s_low;
  const int p = blockIdx.x, l = p / B, b = p - l * B, tid = threadIdx.x;
  const int T = off.o[B], t0 = off.o[b], Tb = off.o[b + 1] - t0;
  long long* oi = indices + (long long)l * 2 * T + t0;
  long long* oj = oi + T;
  for (int k = tid; k < Tb; k += blockDim.x) oi[k] = oj[k] = -1;
  if (Tb == 0) return;                                     // linear_sum_assignment of a [Q, 0] matrix: empty
  const float* C = cost + (long long)l * Q * T + (long long)Q * t0;
  int bad = 0;
  for (int e = tid; e < Q * Tb; e += blockDim.x) {
    const float c = C[e];
    if (c != c || c == -INFINITY) bad = 1;
  }
  if (__syncthreads_or(bad)) {
    if (tid == 0) status[p] = 1;
    return;
  }
  const bool tr = Tb < Q;                                  // a tall matrix is solved transposed
  const int nr = tr ? Tb : Q, nc = tr ? Q : Tb;
  for (int i = tid; i < nr; i += blockDim.x) { u[i] = 0.0; col4row[i] = -1; }
  for (int j = tid; j < nc; j += blockDim.x) { v[j] = 0.0; path[j] = -1; row4col[j] = -1; }
  for (int cur = 0; cur < nr; ++cur) {
    for (int i = tid; i < nr; i += blockDim.x) SR[i] = false;
    for (int j = tid; j < nc; j += blockDim.x) {
      remaining[j] = (short)(nc - j - 1);
      SC[j] = false;
      spc[j] = INFINITY;
    }
    __syncthreads();
    double minVal = 0.0;
    int i = cur, nrem = nc, sink = -1;
    while (sink == -1) {
      if (tid == 0) SR[i] = true;
      const double ui = u[i];
      Pick best{INFINITY, -1, 0};
      for (int it = tid; it < nrem; it += blockDim.x) {
        const int j = remaining[it];
        const float c = tr ? C[(long long)j * Tb + i] : C[(long long)i * Tb + j];
        const double r = __dsub_rn(__dsub_rn(__dadd_rn(minVal, (double)c), ui), v[j]);
        double sj = spc[j];
        if (r < sj) { path[j] = (short)i; spc[j] = sj = r; }
        const Pick cand{sj, it, row4col[j] == -1 ? 1 : 0};
        if (pick_better(cand, best)) best = cand;
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        Pick other{__shfl_xor_sync(0xffffffffu, best.v, o), __shfl_xor_sync(0xffffffffu, best.it, o),
                   __shfl_xor_sync(0xffffffffu, best.free_, o)};
        if (pick_better(other, best)) best = other;
      }
      if ((tid & 31) == 0) wbest[tid >> 5] = best;
      __syncthreads();
      if (tid == 0) {
        Pick bb = wbest[0];
        for (int w = 1; w < LSA_THREADS / 32; ++w)
          if (pick_better(wbest[w], bb)) bb = wbest[w];
        s_low = bb.it < 0 ? INFINITY : bb.v;
        s_index = bb.it;
      }
      __syncthreads();
      minVal = s_low;
      if (minVal == INFINITY) {                            // no finite complete assignment
        if (tid == 0) status[p] = 2;
        return;
      }
      const int index = s_index, j = remaining[index];
      if (row4col[j] == -1) sink = j; else i = row4col[j];
      __syncthreads();                                     // everyone has read remaining[index] and row4col[j]
      if (tid == 0) { SC[j] = true; remaining[index] = remaining[nrem - 1]; }
      --nrem;
      __syncthreads();
    }
    // dual updates
    for (int r = tid; r < nr; r += blockDim.x)
      if (r == cur) u[r] = __dadd_rn(u[r], minVal);
      else if (SR[r]) u[r] = __dadd_rn(u[r], __dsub_rn(minVal, spc[col4row[r]]));
    for (int j = tid; j < nc; j += blockDim.x)
      if (SC[j]) v[j] = __dsub_rn(v[j], __dsub_rn(minVal, spc[j]));
    __syncthreads();
    if (tid == 0) {                                        // augment the previous solution along the path
      int j = sink;
      while (true) {
        const int r = path[j];
        row4col[j] = (short)r;
        const int t = col4row[r];
        col4row[r] = (short)j;
        j = t;
        if (r == cur) break;
      }
    }
    __syncthreads();
  }
  if (!tr) {
    for (int r = tid; r < nr; r += blockDim.x) { oi[r] = r; oj[r] = col4row[r]; }
  } else {                                                 // argsort of col4row: queries ascending
    for (int r = tid; r < nr; r += blockDim.x) {
      const int c = col4row[r];
      int rank = 0;
      for (int k = 0; k < nr; ++k) rank += col4row[k] < c;
      oi[rank] = c;
      oj[rank] = r;
    }
  }
}

__device__ __forceinline__ double block_sum(double x, double* sh) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = x;
  __syncthreads();
  double t = 0.0;
  for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += sh[w];
  return t;
}

// Grid L.  out[l] = {loss_ce, class_error, loss_bbox, loss_giou, cardinality_error}.
__global__ void __launch_bounds__(LOSS_THREADS) set_losses_kernel(
    Layers lay, int B, int Q, int C1, const long long* __restrict__ tgt_ids, const float* __restrict__ tgt_boxes, Offsets off,
    const long long* __restrict__ indices, const float* __restrict__ empty_weight, const float* __restrict__ num_boxes,
    float* __restrict__ out) {
  __shared__ double sh[LOSS_THREADS / 32];
  __shared__ int card[CRIT_MAX_IMAGES], correct;
  const int l = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int T = off.o[B];
  const long long* ii = indices + (long long)l * 2 * T;
  const long long* jj = ii + T;
  for (int b = tid; b < B; b += blockDim.x) card[b] = 0;
  if (tid == 0) correct = 0;
  __syncthreads();
  // cross-entropy with empty_weight, the cardinality count and the matched rows' top-1: one warp per row
  double wnll = 0.0, wsum = 0.0;
  for (int r = warp; r < B * Q; r += LOSS_THREADS / 32) {
    const int b = r / Q, q = r - b * Q;
    const float* x = lay.logits[l] + (long long)r * C1;
    const int t0 = off.o[b], K = min(Q, off.o[b + 1] - t0);
    int k = -1;
    for (int s = 0; s < K && k < 0; s += 32) {
      const unsigned hit = __ballot_sync(0xffffffffu, s + lane < K && ii[t0 + s + lane] == q);
      if (hit) k = s + __ffs(hit) - 1;
    }
    long long tc = C1 - 1;                                  // no-object
    if (k >= 0) {
      const long long j = jj[t0 + k];
      tc = (j >= 0 && j < off.o[b + 1] - t0) ? tgt_ids[t0 + j] : -1;
    }
    float m, s;
    warp_softmax_stats(x, C1, lane, m, s);
    float best = 0.f;
    int bi = -1;
    for (int c = lane; c < C1; c += 32)
      if (argmax_better(x[c], c, best, bi)) { best = x[c]; bi = c; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ob = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (argmax_better(ob, oi, best, bi)) { best = ob; bi = oi; }
    }
    if (lane == 0) {
      const bool valid = tc >= 0 && tc < C1;
      const float w = valid ? empty_weight[tc] : __int_as_float(0x7fc00000);
      const float nll = valid ? -((x[tc] - m) - logf(s)) : __int_as_float(0x7fc00000);
      wnll += (double)w * (double)nll;
      wsum += (double)w;
      if (bi != C1 - 1) atomicAdd(&card[b], 1);
      if (k >= 0 && bi == tc) atomicAdd(&correct, 1);
    }
  }
  // the matched pairs: L1 and 1 - GIoU
  double l1 = 0.0, gi = 0.0;
  for (int b = 0; b < B; ++b) {
    const int t0 = off.o[b], Tb = off.o[b + 1] - t0, K = min(Q, Tb);
    for (int k = tid; k < K; k += blockDim.x) {
      const long long i = ii[t0 + k], j = jj[t0 + k];
      if (i < 0 || i >= Q || j < 0 || j >= Tb) { l1 += NAN; gi += NAN; continue; }
      const float* pb = lay.boxes[l] + ((long long)b * Q + i) * 4;
      const float* tb = tgt_boxes + (t0 + j) * 4;
      for (int c = 0; c < 4; ++c) l1 += (double)fabsf(__fsub_rn(pb[c], tb[c]));
      gi += (double)__fsub_rn(1.f, giou(pb, tb));
    }
  }
  wnll = block_sum(wnll, sh);
  wsum = block_sum(wsum, sh);
  l1 = block_sum(l1, sh);
  gi = block_sum(gi, sh);
  if (tid == 0) {
    const float nb = *num_boxes;
    int matched = 0;
    float card_err = 0.f;
    for (int b = 0; b < B; ++b) {
      const int Tb = off.o[b + 1] - off.o[b];
      matched += min(Q, Tb);
      card_err = __fadd_rn(card_err, fabsf((float)card[b] - (float)Tb));
    }
    float* o = out + l * 5;
    o[0] = (float)(wnll / wsum);
    // misc.accuracy: correct * (100 / batch_size) in fp32; 0 when nothing is matched
    o[1] = matched ? __fsub_rn(100.f, __fmul_rn((float)correct, (float)(100.0 / matched))) : 100.f;
    o[2] = __fdiv_rn((float)l1, nb);
    o[3] = __fdiv_rn((float)gi, nb);
    o[4] = __fdiv_rn(card_err, (float)B);
  }
}

struct MaskImages {
  const void* masks[CRIT_MAX_IMAGES];   // [T_b, H_b, W_b]
  int H[CRIT_MAX_IMAGES], W[CRIT_MAX_IMAGES];
  int first[CRIT_MAX_IMAGES + 1];       // matched masks of images < b
};

__device__ __forceinline__ float target_at(const void* base, int dtype, long long e) {
  return dtype ? static_cast<const float*>(base)[e] : (float)static_cast<const uint8_t*>(base)[e];
}

// Grid (ceil(Hm / MASK_ROWS), masks).  Shared: the [h, w] plane, then per target column the packed taps and the weight.
__global__ void __launch_bounds__(MASK_THREADS) mask_partials_kernel(
    const float* __restrict__ pred, int B, int Q, int h, int w, int Hm, int Wm, MaskImages im, int dtype, Offsets off,
    const long long* __restrict__ indices, double* __restrict__ partials) {
  extern __shared__ float smem[];
  __shared__ double sh[MASK_THREADS / 32];
  const int mk = blockIdx.y, y0 = blockIdx.x * MASK_ROWS, tid = threadIdx.x;
  int b = 0;
  while (mk >= im.first[b + 1]) ++b;
  const int T = off.o[B], t0 = off.o[b], k = mk - im.first[b];
  const long long i = indices[t0 + k], j = indices[T + t0 + k];
  double acc[4] = {0.0, 0.0, 0.0, 0.0};
  const bool ok = i >= 0 && i < Q && j >= 0 && j < off.o[b + 1] - t0;
  float* P = smem;
  int* ctap = reinterpret_cast<int*>(P + h * w);
  float* cl1 = reinterpret_cast<float*>(ctap + Wm);
  const bool copy = h == Hm && w == Wm;                       // F.interpolate to the same size copies
  if (ok) {
    const float* src = pred + ((long long)b * Q + i) * h * w;
    for (int e = tid; e < h * w; e += blockDim.x) P[e] = src[e];
    const float bw = (float)w / (float)Wm;
    for (int x = tid; x < Wm; x += blockDim.x) {
      int a = x, c = x;
      float l1 = 0.f;
      if (!copy) linear_taps(x, bw, w, a, c, l1);
      ctap[x] = a | (c << 16);
      cl1[x] = l1;
    }
  }
  __syncthreads();
  if (ok) {
    const float bh = (float)h / (float)Hm;
    const int Hb = im.H[b], Wb = im.W[b];
    const long long plane = j * (long long)Hb * Wb;
    const int rows = min(MASK_ROWS, Hm - y0);
    for (int e = tid; e < rows * Wm; e += blockDim.x) {
      const int r = e / Wm, x = e - r * Wm, y = y0 + r;
      int ya = y, yb = y;
      float lh1 = 0.f;
      if (!copy) linear_taps(y, bh, h, ya, yb, lh1);
      const int cx = ctap[x], x0 = cx & 0xffff, x1 = cx >> 16;
      float v;
      if (copy) {
        v = P[ya * w + x0];
      } else {
        const float lw1 = cl1[x], lw0 = 1.f - lw1, lh0 = 1.f - lh1;
        v = lh0 * (lw0 * P[ya * w + x0] + lw1 * P[ya * w + x1]) + lh1 * (lw0 * P[yb * w + x0] + lw1 * P[yb * w + x1]);
      }
      const float t = (y < Hb && x < Wb) ? target_at(im.masks[b], dtype, plane + (long long)y * Wb + x) : 0.f;
      const float prob = 1.f / (1.f + expf(-v));
      // F.binary_cross_entropy_with_logits: (1 - t) x - log_sigmoid(x)
      const float ls = (v != v ? v : fminf(v, 0.f)) - log1pf(expf(-fabsf(v)));
      const float ce = (1.f - t) * v - ls;
      const float pt = prob * t + (1.f - prob) * (1.f - t);
      const float f = (0.25f * t + 0.75f * (1.f - t)) * (ce * ((1.f - pt) * (1.f - pt)));
      acc[0] += (double)f;
      acc[1] += (double)(prob * t);
      acc[2] += (double)prob;
      acc[3] += (double)t;
    }
  }
  double* o = partials + ((long long)mk * gridDim.x + blockIdx.x) * 4;
  for (int c = 0; c < 4; ++c) {
    const double s = block_sum(acc[c], sh);
    if (tid == 0) o[c] = ok ? s : NAN;
  }
}

// One CTA: per mask (thread) the fixed-order sum over the row chunks, then the masks in order.
__global__ void mask_finish_kernel(const double* __restrict__ partials, int masks, int chunks, long long pixels,
                                   const float* __restrict__ num_boxes, double* __restrict__ per_mask, float* __restrict__ out) {
  for (int mk = threadIdx.x; mk < masks; mk += blockDim.x) {
    double s[4] = {0.0, 0.0, 0.0, 0.0};
    for (int c = 0; c < chunks; ++c)
      for (int k = 0; k < 4; ++k) s[k] += partials[((long long)mk * chunks + c) * 4 + k];
    per_mask[2 * mk] = (double)(float)(s[0] / (double)pixels);                 // loss.mean(1)
    per_mask[2 * mk + 1] = 1.0 - (2.0 * s[1] + 1.0) / (s[2] + s[3] + 1.0);     // dice_loss
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double f = 0.0, d = 0.0;
    for (int mk = 0; mk < masks; ++mk) { f += per_mask[2 * mk]; d += per_mask[2 * mk + 1]; }
    const float nb = *num_boxes;
    out[0] = __fdiv_rn((float)f, nb);
    out[1] = __fdiv_rn((float)d, nb);
  }
}

int fill_offsets(Offsets& off, int B, const int* offsets) {
  MMX_REQUIRE(offsets && B > 0 && B <= CRIT_MAX_IMAGES, "1 - 64 images per call, with their target offsets");
  MMX_REQUIRE(offsets[0] == 0, "target offsets start at 0");
  for (int b = 0; b <= B; ++b) {
    if (b) MMX_REQUIRE(offsets[b] >= offsets[b - 1], "target offsets must not decrease");
    off.o[b] = offsets[b];
  }
  return 0;
}

int fill_layers(Layers& lay, int L, const float* const* logits, const float* const* boxes) {
  MMX_REQUIRE(L > 0 && L <= CRIT_MAX_LAYERS, "1 - 16 decoder layers per call");
  MMX_REQUIRE(logits && boxes, "bad arguments");
  for (int l = 0; l < L; ++l) {
    MMX_REQUIRE(logits[l] && boxes[l], "every layer needs pred_logits and pred_boxes");
    lay.logits[l] = logits[l];
    lay.boxes[l] = boxes[l];
  }
  return 0;
}

}  // namespace
}  // namespace mmx

using namespace mmx;
extern "C" {

int mmx_detr_match_cost(const float* const* logits, const float* const* boxes, int L, int B, int Q, int C1,
                        const int64_t* tgt_ids, const float* tgt_boxes, const int* tgt_offsets, float w_class, float w_bbox,
                        float w_giou, float* cost, int* status, void* stream) {
  Layers lay;
  Offsets off;
  MMX_TRY(fill_layers(lay, L, logits, boxes));
  MMX_TRY(fill_offsets(off, B, tgt_offsets));
  MMX_REQUIRE(Q > 0 && C1 >= 2 && status, "bad arguments");
  MMX_REQUIRE(off.o[B] == 0 || (tgt_ids && tgt_boxes && cost), "targets and the cost buffer are needed");
  MMX_REQUIRE((long long)L * Q * off.o[B] < (1ll << 31), "cost matrix too large");
  cudaStream_t st = (cudaStream_t)stream;
  MMX_CHECK_CUDA(cudaMemsetAsync(status, 0, sizeof(int) * L, st));
  match_cost_kernel<<<dim3(cdiv(Q, COST_WARPS), B, L), COST_WARPS * 32, 0, st>>>(
      lay, B, Q, C1, reinterpret_cast<const long long*>(tgt_ids), tgt_boxes, off, w_class, w_bbox, w_giou, cost, status);
  MMX_LAUNCH_CHECK();
  return 0;
}

int mmx_detr_match_lsa(const float* cost, int L, int B, int Q, const int* tgt_offsets, int64_t* indices, int* status,
                       void* stream) {
  Offsets off;
  MMX_TRY(fill_offsets(off, B, tgt_offsets));
  MMX_REQUIRE(L > 0 && Q > 0 && status, "bad arguments");
  MMX_REQUIRE(Q <= LSA_MAX, "at most 1024 rows (queries) per assignment problem");
  for (int b = 0; b < B; ++b) MMX_REQUIRE(off.o[b + 1] - off.o[b] <= LSA_MAX, "at most 1024 columns (targets) per problem");
  MMX_REQUIRE(off.o[B] == 0 || (cost && indices), "bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  MMX_CHECK_CUDA(cudaMemsetAsync(status, 0, sizeof(int) * L * B, st));
  if (off.o[B] == 0) return 0;
  lsa_kernel<<<L * B, LSA_THREADS, 0, st>>>(cost, B, Q, off, reinterpret_cast<long long*>(indices), status);
  MMX_LAUNCH_CHECK();
  return 0;
}

int mmx_detr_set_losses(const float* const* logits, const float* const* boxes, int L, int B, int Q, int C1,
                        const int64_t* tgt_ids, const float* tgt_boxes, const int* tgt_offsets, const int64_t* indices,
                        const float* empty_weight, const float* num_boxes, float* out, void* stream) {
  Layers lay;
  Offsets off;
  MMX_TRY(fill_layers(lay, L, logits, boxes));
  MMX_TRY(fill_offsets(off, B, tgt_offsets));
  MMX_REQUIRE(Q > 0 && C1 >= 2 && empty_weight && num_boxes && out, "bad arguments");
  MMX_REQUIRE(off.o[B] == 0 || (tgt_ids && tgt_boxes && indices), "bad arguments");
  set_losses_kernel<<<L, LOSS_THREADS, 0, (cudaStream_t)stream>>>(
      lay, B, Q, C1, reinterpret_cast<const long long*>(tgt_ids), tgt_boxes, off, reinterpret_cast<const long long*>(indices),
      empty_weight, num_boxes, out);
  MMX_LAUNCH_CHECK();
  return 0;
}

int mmx_detr_mask_losses(const float* pred_masks, int B, int Q, int h, int w, const void* const* tgt_masks, const int* tgt_hw,
                         int mask_dtype, const int* tgt_offsets, const int64_t* indices, const float* num_boxes, float* out,
                         void* stream) {
  Offsets off;
  MMX_TRY(fill_offsets(off, B, tgt_offsets));
  MMX_REQUIRE(pred_masks && tgt_masks && tgt_hw && num_boxes && out && Q > 0 && h > 0 && w > 0, "bad arguments");
  MMX_REQUIRE(mask_dtype == 0 || mask_dtype == 1, "target masks are uint8 / bool (0) or float32 (1)");
  MMX_REQUIRE(h < 65536 && w < 65536, "mask plane too large");
  MaskImages im;
  int Hm = 0, Wm = 0, n = 0;
  for (int b = 0; b < B; ++b) {
    const int Tb = off.o[b + 1] - off.o[b];
    im.masks[b] = tgt_masks[b];
    im.H[b] = tgt_hw[2 * b];
    im.W[b] = tgt_hw[2 * b + 1];
    MMX_REQUIRE(im.H[b] >= 0 && im.W[b] >= 0 && (Tb == 0 || tgt_masks[b]), "bad target masks");
    im.first[b] = n;
    n += min(Q, Tb);
    Hm = max(Hm, im.H[b]);
    Wm = max(Wm, im.W[b]);
  }
  im.first[B] = n;
  MMX_REQUIRE(Wm < 65536, "target masks too wide");
  cudaStream_t st = (cudaStream_t)stream;
  if (n == 0 || Hm == 0 || Wm == 0) {
    MMX_CHECK_CUDA(cudaMemsetAsync(out, 0, 2 * sizeof(float), st));
    return 0;
  }
  MMX_REQUIRE(indices, "bad arguments");
  const int chunks = cdiv(Hm, MASK_ROWS);
  const size_t smem = (size_t)h * w * sizeof(float) + (size_t)Wm * 8;
  MMX_REQUIRE(smem <= 200 * 1024, "mask plane plus the per-column taps exceed shared memory");
  if (smem > 48 * 1024)
    MMX_CHECK_CUDA(cudaFuncSetAttribute(mask_partials_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  keep_stream_scratch_cached();
  double* partials = nullptr;
  const size_t bytes = ((size_t)n * chunks * 4 + (size_t)n * 2) * sizeof(double);
  MMX_CHECK_CUDA(cudaMallocAsync(&partials, bytes, st));
  mask_partials_kernel<<<dim3(chunks, n), MASK_THREADS, smem, st>>>(pred_masks, B, Q, h, w, Hm, Wm, im, mask_dtype, off,
                                                                      reinterpret_cast<const long long*>(indices), partials);
  MMX_LAUNCH_CHECK();
  mask_finish_kernel<<<1, 256, 0, st>>>(partials, n, chunks, (long long)Hm * Wm, num_boxes, partials + (size_t)n * chunks * 4,
                                        out);
  MMX_LAUNCH_CHECK();
  MMX_CHECK_CUDA(cudaFreeAsync(partials, st));
  return 0;
}
}
