// YOLOv3 training loss (forward + gradient w.r.t. the raw logits), one scale per call.
// Replaces model.py:192-304 (loss_layer: dozens of elementwise TF ops + a serial
// per-image tf.while_loop for the ignore mask) and model.py:307-345 (box_iou), and the
// part of TF autodiff that differentiates them (train.py:112).
//
//   1. loss_gather_gt_kernel : per image, compact the ground-truth boxes of this scale
//      (cells with object_mask == 1, model.py:224) into a list.
//   2. loss_kernel : one WARP per predicted box (n, h, w, anchor).  Lanes read the 5+C
//      logits and the 5+C+1 y_true values of the box coalesced, decode the box
//      (model.py:82-137), scan the image's gt list for the best IoU (ignore mask,
//      model.py:220-239), evaluate the four loss terms (model.py:248-302) and, if asked,
//      write d(total)/d(logit) — the formulas of SURVEY.md Appendix B.3.
// HBM-bound: reads fm (3.62 MB/img @416) + y_true (3.66 MB/img), writes the gradient.
#include "common.cuh"

namespace yb {

struct LossParams {
  const float* fm;       // [n, gh, gw, 3*E]
  const float* y_true;   // [n, gh, gw, 3, E+1]
  int n, gh, gw, C, E;
  float ratio_h, ratio_w, img_h, img_w;
  float anchor_w[3], anchor_h[3];
  int label_smooth, focal;
  float inv_n;           // 1 / batch size (model.py:206)
  float grad_mul;        // inv_n * loss_scale: what the stored gradient is multiplied by (fp16 storage needs loss scaling)
  const float* gt_boxes; // [n, cap, 4] cx,cy,w,h
  const int* gt_count;   // [n]
  int cap;
  double* loss4;         // xy, wh, conf, class (accumulated)
  void* dfm;             // nullable gradient output
  int dfm_dtype;         // YB_F32: same layout as fm; YB_F16/YB_BF16: [rows, dfm_ld], rows = n*gh*gw, cols 3*E (+ zero pad)
  int dfm_ld;
};

__global__ void loss_gather_gt_kernel(const float* __restrict__ y_true, int n, int cells3, int E1,
                                      float* __restrict__ gt_boxes, int* __restrict__ gt_count) {
  const int img = blockIdx.y;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < cells3; i += gridDim.x * blockDim.x) {
    const float* row = y_true + ((long)img * cells3 + i) * E1;
    if (row[4] != 0.f) {   // tf.cast(object_mask, 'bool')
      const int slot = atomicAdd(&gt_count[img], 1);
      float4 b = make_float4(row[0], row[1], row[2], row[3]);
      reinterpret_cast<float4*>(gt_boxes)[(long)img * cells3 + slot] = b;
    }
  }
}

__device__ __forceinline__ float sigmoid_f(float x) { return 1.0f / (1.0f + expf(-x)); }
// [TF] sigmoid_cross_entropy_with_logits: max(z,0) - z*y + log(1+exp(-|z|))
__device__ __forceinline__ float bce_logits(float z, float y) { return fmaxf(z, 0.f) - z * y + log1pf(expf(-fabsf(z))); }

template <typename T>
__device__ __forceinline__ void store_grad(const LossParams& p, long box, int a, long cellrow, int j, float g) {
  if (p.dfm_dtype == YB_F32) {
    static_cast<float*>(p.dfm)[box * p.E + j] = g;
  } else {
    static_cast<T*>(p.dfm)[cellrow * p.dfm_ld + a * p.E + j] = static_cast<T>(g);
  }
}

template <typename T>
__global__ void __launch_bounds__(256) loss_kernel(const LossParams p) {
  __shared__ double s_sum[8][4];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const long nbox = (long)p.n * p.gh * p.gw * 3;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  for (long box = (long)blockIdx.x * 8 + wib; box < nbox; box += (long)gridDim.x * 8) {
    const int a = (int)(box % 3);
    const long cellrow = box / 3;                      // (n, h, w) flattened
    const int cell = (int)(cellrow % ((long)p.gh * p.gw));
    const int img = (int)(cellrow / ((long)p.gh * p.gw));
    const float* lrow = p.fm + box * p.E;
    const float* yrow = p.y_true + box * (p.E + 1);
    // lanes 0..4 fetch the box / conf logits and targets; broadcast
    const float lv = lane < 5 ? lrow[lane] : 0.f;
    const float yv = lane < 5 ? yrow[lane] : 0.f;
    const float tx = __shfl_sync(0xffffffffu, lv, 0), ty = __shfl_sync(0xffffffffu, lv, 1);
    const float tw = __shfl_sync(0xffffffffu, lv, 2), th = __shfl_sync(0xffffffffu, lv, 3);
    const float tc = __shfl_sync(0xffffffffu, lv, 4);
    const float gx = __shfl_sync(0xffffffffu, yv, 0), gy = __shfl_sync(0xffffffffu, yv, 1);
    const float gw_ = __shfl_sync(0xffffffffu, yv, 2), gh_ = __shfl_sync(0xffffffffu, yv, 3);
    const float m = __shfl_sync(0xffffffffu, yv, 4);
    const float mix = yrow[p.E];                        // broadcast load
    // ---- decode (model.py:105-126) ----
    const float offx = (float)(cell % p.gw), offy = (float)(cell / p.gw);
    const float sx = sigmoid_f(tx), sy = sigmoid_f(ty);
    const float pcx = (sx + offx) * p.ratio_w, pcy = (sy + offy) * p.ratio_h;
    const float ew = expf(tw), eh = expf(th);
    const float pw = ew * (p.anchor_w[a] / p.ratio_w) * p.ratio_w;
    const float ph = eh * (p.anchor_h[a] / p.ratio_h) * p.ratio_h;
    // ---- ignore mask: best IoU against this image's gt boxes (model.py:220-239, 307-345) ----
    const int cnt = p.gt_count[img];
    float best = -3.4e38f;                              // [TF] reduce_max over an empty axis
    {
      const float4* gl = reinterpret_cast<const float4*>(p.gt_boxes) + (long)img * p.cap;
      const float px0 = pcx - pw / 2.f, px1 = pcx + pw / 2.f, py0 = pcy - ph / 2.f, py1 = pcy + ph / 2.f;
      const float parea = pw * ph;
      for (int j = lane; j < cnt; j += 32) {
        const float4 g = __ldg(gl + j);
        const float ix = fmaxf(fminf(px1, g.x + g.z / 2.f) - fmaxf(px0, g.x - g.z / 2.f), 0.f);
        const float iy = fmaxf(fminf(py1, g.y + g.w / 2.f) - fmaxf(py0, g.y - g.w / 2.f), 0.f);
        const float inter = ix * iy;
        best = fmaxf(best, inter / (parea + g.z * g.w - inter + 1e-10f));
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) best = fmaxf(best, __shfl_xor_sync(0xffffffffu, best, o));
    }
    const float ignore = best < 0.5f ? 1.f : 0.f;
    // ---- box terms (lane 0 computes, model.py:248-277) ----
    const float scale = 2.f - (gw_ / p.img_w) * (gh_ / p.img_h);
    const float cbox = m * scale * mix;
    const float true_x = gx / p.ratio_w - offx, true_y = gy / p.ratio_h - offy;
    const float pred_x = pcx / p.ratio_w - offx, pred_y = pcy / p.ratio_h - offy;
    float ttw = gw_ / p.anchor_w[a], tth = gh_ / p.anchor_h[a];
    float ptw = pw / p.anchor_w[a], pth = ph / p.anchor_h[a];
    const bool pw_zero = ptw == 0.f, ph_zero = pth == 0.f;
    if (ttw == 0.f) ttw = 1.f;
    if (tth == 0.f) tth = 1.f;
    if (pw_zero) ptw = 1.f;
    if (ph_zero) pth = 1.f;
    const bool w_in = ptw > 1e-9f && ptw < 1e9f, h_in = pth > 1e-9f && pth < 1e9f;
    const float ltw = logf(fminf(fmaxf(ttw, 1e-9f), 1e9f)), lth = logf(fminf(fmaxf(tth, 1e-9f), 1e9f));
    const float lpw = logf(fminf(fmaxf(ptw, 1e-9f), 1e9f)), lph = logf(fminf(fmaxf(pth, 1e-9f), 1e9f));
    const float dx = true_x - pred_x, dy = true_y - pred_y, dw = ltw - lpw, dh = lth - lph;
    // ---- conf (model.py:280-292) ----
    const float sc = sigmoid_f(tc);
    const float bce_c = bce_logits(tc, m);
    const float wconf = m + (1.f - m) * ignore;
    const float fm_ = m - sc;
    const float focal = p.focal ? fm_ * fm_ : 1.f;
    if (lane == 0) {
      acc[0] += (dx * dx + dy * dy) * cbox;
      acc[1] += (dw * dw + dh * dh) * cbox;
      acc[2] += wconf * bce_c * focal * mix;
    }
    if (p.dfm != nullptr && lane < 5) {
      float g;
      const float cg = cbox * p.grad_mul;
      if (lane == 0) g = -2.f * dx * sx * (1.f - sx) * cg;
      else if (lane == 1) g = -2.f * dy * sy * (1.f - sy) * cg;
      else if (lane == 2) g = (w_in && !pw_zero) ? -2.f * dw * cg : 0.f;
      else if (lane == 3) g = (h_in && !ph_zero) ? -2.f * dh * cg : 0.f;
      else {
        const float gc = wconf * mix * p.grad_mul;
        g = p.focal ? gc * (fm_ * fm_ * (sc - m) - 2.f * fm_ * sc * (1.f - sc) * bce_c) : gc * (sc - m);
      }
      store_grad<T>(p, box, a, cellrow, lane, g);
    }
    // ---- class term (model.py:296-302) ----
    float cls = 0.f;
    if (m == 0.f) {
      // no object in this (cell, anchor) — all but a few hundred of the 10^5 boxes: the class loss and its gradient are
      // object_mask * (...) = 0, so neither the 2 x C logits / targets are read nor C sigmoids evaluated (the kernel was
      // latency-bound on exactly that loop)
      if (p.dfm != nullptr)
        for (int k = lane; k < p.C; k += 32) store_grad<T>(p, box, a, cellrow, 5 + k, 0.f);
      continue;
    }
    for (int k = lane; k < p.C; k += 32) {
      const float z = lrow[5 + k];
      float t = yrow[5 + k];
      if (p.label_smooth) t = (1.f - 0.01f) * t + 0.01f * 1.f / (float)p.C;
      if (m != 0.f) cls += bce_logits(z, t);
      if (p.dfm != nullptr) store_grad<T>(p, box, a, cellrow, 5 + k, m * mix * (sigmoid_f(z) - t) * p.grad_mul);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) cls += __shfl_xor_sync(0xffffffffu, cls, o);
    if (lane == 0) acc[3] += m * cls * mix;
  }
  if (lane == 0)
    for (int i = 0; i < 4; ++i) s_sum[wib][i] = (double)acc[i];
  __syncthreads();
  if (threadIdx.x < 4) {
    double t = 0.0;
    for (int w = 0; w < 8; ++w) t += s_sum[w][threadIdx.x];
    atomicAdd(p.loss4 + threadIdx.x, t * (double)p.inv_n);
  }
}

// zero the padding columns [3E, ld) of a 16-bit gradient buffer
template <typename T>
__global__ void loss_pad_kernel(T* dfm, long rows, int used, int ld) {
  const int padw = ld - used;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < rows * padw; i += (long)gridDim.x * blockDim.x)
    dfm[(i / padw) * ld + used + (i % padw)] = static_cast<T>(0.f);
}

__global__ void box_iou_kernel(const float* __restrict__ pred, const float* __restrict__ gt, long P, int V,
                               float* __restrict__ out) {
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < P * V; i += (long)gridDim.x * blockDim.x) {
    const float4 a = reinterpret_cast<const float4*>(pred)[i / V];
    const float4 g = reinterpret_cast<const float4*>(gt)[i % V];
    const float ix = fmaxf(fminf(a.x + a.z / 2.f, g.x + g.z / 2.f) - fmaxf(a.x - a.z / 2.f, g.x - g.z / 2.f), 0.f);
    const float iy = fmaxf(fminf(a.y + a.w / 2.f, g.y + g.w / 2.f) - fmaxf(a.y - a.w / 2.f, g.y - g.w / 2.f), 0.f);
    const float inter = ix * iy;
    out[i] = inter / (a.z * a.w + g.z * g.w - inter + 1e-10f);
  }
}

}  // namespace yb

using namespace yb;

extern "C" int yb_loss_workspace_bytes(int n, int gh, int gw, size_t* bytes) {
  YB_REQUIRE(bytes && n > 0 && gh > 0 && gw > 0, "loss_workspace: bad argument");
  *bytes = (size_t)n * gh * gw * 3 * 16 + ((size_t)n * 4 + 255) / 256 * 256;
  return YB_OK;
}

extern "C" int yb_loss_layer(const float* feature_map, const float* y_true, int n, int gh, int gw, int img_h, int img_w,
                             int class_num, const float* anchors3x2, int use_label_smooth, int use_focal_loss,
                             float inv_batch, float loss_scale, void* workspace, size_t workspace_bytes, double* loss4,
                             void* dfm, int dfm_dtype, int dfm_ld, void* stream) {
  YB_REQUIRE(feature_map && y_true && anchors3x2 && workspace && loss4, "loss_layer: null pointer");
  YB_REQUIRE(n > 0 && gh > 0 && gw > 0 && class_num > 0, "loss_layer: bad shape");
  size_t need = 0;
  yb_loss_workspace_bytes(n, gh, gw, &need);
  if (workspace_bytes < need) { set_error("loss_layer: workspace too small (%zu < %zu)", workspace_bytes, need); return YB_ERR_WORKSPACE; }
  YB_REQUIRE(((uintptr_t)workspace & 15) == 0, "loss_layer: workspace must be 16-byte aligned");
  const int E = 5 + class_num;
  if (dfm) {
    YB_REQUIRE(dfm_dtype == YB_F32 || dfm_dtype == YB_F16 || dfm_dtype == YB_BF16, "loss_layer: bad dfm dtype");
    YB_REQUIRE(dfm_dtype == YB_F32 || dfm_ld >= 3 * E, "loss_layer: dfm_ld %d < %d", dfm_ld, 3 * E);
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int cells3 = gh * gw * 3;
  int* gt_count = reinterpret_cast<int*>(workspace);
  float* gt_boxes = reinterpret_cast<float*>(static_cast<uint8_t*>(workspace) + ((size_t)n * 4 + 255) / 256 * 256);
  YB_CUDA(cudaMemsetAsync(gt_count, 0, (size_t)n * 4, st));
  dim3 g1(ceil_div(cells3, 256) < 64 ? ceil_div(cells3, 256) : 64, n);
  loss_gather_gt_kernel<<<g1, 256, 0, st>>>(y_true, n, cells3, E + 1, gt_boxes, gt_count);
  YB_CUDA(cudaGetLastError());
  LossParams p;
  p.fm = feature_map; p.y_true = y_true; p.n = n; p.gh = gh; p.gw = gw; p.C = class_num; p.E = E;
  p.ratio_h = (float)((double)img_h / gh); p.ratio_w = (float)((double)img_w / gw);
  p.img_h = (float)img_h; p.img_w = (float)img_w;
  for (int i = 0; i < 3; ++i) { p.anchor_w[i] = anchors3x2[2 * i]; p.anchor_h[i] = anchors3x2[2 * i + 1]; }
  p.label_smooth = use_label_smooth; p.focal = use_focal_loss; p.inv_n = inv_batch;
  p.grad_mul = inv_batch * (loss_scale > 0.f ? loss_scale : 1.f);
  p.gt_boxes = gt_boxes; p.gt_count = gt_count; p.cap = cells3; p.loss4 = loss4;
  p.dfm = dfm; p.dfm_dtype = dfm_dtype; p.dfm_ld = dfm_ld;
  const long nbox = (long)n * cells3;
  long blocks = (nbox + 7) / 8;
  const long capb = (long)num_sms() * 16;
  if (blocks > capb) blocks = capb;
  if (dfm && dfm_dtype == YB_BF16) {
    loss_kernel<__nv_bfloat16><<<(int)blocks, 256, 0, st>>>(p);
    if (dfm_ld > 3 * E) loss_pad_kernel<__nv_bfloat16><<<256, 256, 0, st>>>(static_cast<__nv_bfloat16*>(dfm), (long)n * gh * gw, 3 * E, dfm_ld);
  } else {
    loss_kernel<__half><<<(int)blocks, 256, 0, st>>>(p);
    if (dfm && dfm_dtype == YB_F16 && dfm_ld > 3 * E)
      loss_pad_kernel<__half><<<256, 256, 0, st>>>(static_cast<__half*>(dfm), (long)n * gh * gw, 3 * E, dfm_ld);
  }
  YB_CUDA(cudaGetLastError());
  return YB_OK;
}

__global__ void loss_finalize_kernel(const double* l4, float* out5) {
  if (threadIdx.x == 0) {
    const double t = l4[0] + l4[1] + l4[2] + l4[3];
    out5[0] = (float)t; out5[1] = (float)l4[0]; out5[2] = (float)l4[1]; out5[3] = (float)l4[2]; out5[4] = (float)l4[3];
  }
}

extern "C" int yb_loss_finalize(const double* loss4, float* out5, void* stream) {
  YB_REQUIRE(loss4 && out5, "loss_finalize: null pointer");
  loss_finalize_kernel<<<1, 32, 0, static_cast<cudaStream_t>(stream)>>>(loss4, out5);
  YB_CUDA(cudaGetLastError());
  return YB_OK;
}

extern "C" int yb_box_iou(const float* pred_boxes, const float* true_boxes, long num_pred, int num_true, float* iou,
                          void* stream) {
  YB_REQUIRE(num_pred >= 0 && num_true >= 0, "box_iou: bad shape");
  if (num_pred == 0 || num_true == 0) return YB_OK;
  YB_REQUIRE(pred_boxes && true_boxes && iou, "box_iou: null pointer");
  const long total = num_pred * num_true;
  long g = (total + 255) / 256;
  if (g > 148L * 32) g = 148L * 32;
  box_iou_kernel<<<(int)g, 256, 0, static_cast<cudaStream_t>(stream)>>>(pred_boxes, true_boxes, num_pred, num_true, iou);
  YB_CUDA(cudaGetLastError());
  return YB_OK;
}
