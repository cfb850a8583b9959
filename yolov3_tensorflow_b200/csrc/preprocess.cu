// The two host-side steps either side of the hot path, moved onto the device (SURVEY.md 8f N3):
//   * process_box (utils/data_utils.py:51-115): ground-truth box lists -> the three y_true tensors consumed by
//     loss_layer.  The reference builds 3.66 MB per 416x416 image in numpy and ships it host -> device; here only the
//     box lists (<= 50 x 24 B per image) cross PCIe and the tensors are produced at HBM speed.
//   * letterbox_resize + BGR->RGB + /255 (utils/data_aug.py:274-293, test_single_image.py:39-46): uint8 BGR image ->
//     float32 RGB network input, nearest-neighbour (the reference's interp=0) with the 128-grey border; for a batch
//     (yb_resize_batch) nearest or bilinear, and for the training resize (yb_resize_batch_interp) every cv2.resize
//     interpolation the reference draws, 0..4, one per image, from per-image tap tables built on the host.
// Both are bit-exact restatements: float32 operations in the reference's order (__f*_rn: no FMA contraction), the
// resize index in double like OpenCV's resizeNN.
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstring>

#include "common.cuh"

namespace yb {

// y_true[..., :] = 0 and y_true[..., -1] = 1 (utils/data_utils.py:72-79) for the three scales in one launch:
// float4 stores over each tensor's multiple-of-4 prefix, the <= 3 trailing floats by one thread.
__global__ void __launch_bounds__(256) ytrue_fill_kernel(float* __restrict__ y1, long n1, float* __restrict__ y2, long n2,
                                                          float* __restrict__ y3, long n3, int E1 /* 6 + C */) {
  const long q1 = n1 / 4, q2 = n2 / 4, q3 = n3 / 4;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < q1 + q2 + q3; i += (long)gridDim.x * blockDim.x) {
    long e;
    float* dst;
    if (i < q1) { e = i * 4; dst = y1 + e; }
    else if (i < q1 + q2) { e = (i - q1) * 4; dst = y2 + e; }
    else { e = (i - q1 - q2) * 4; dst = y3 + e; }
    const int m = (int)(e % E1);                 // position of the first of the 4 elements inside its box record
    float4 v;                                    // the record's last element (mix-up weight) is the only 1
    v.x = ((m + 0) % E1 == E1 - 1) ? 1.f : 0.f;
    v.y = ((m + 1) % E1 == E1 - 1) ? 1.f : 0.f;
    v.z = ((m + 2) % E1 == E1 - 1) ? 1.f : 0.f;
    v.w = ((m + 3) % E1 == E1 - 1) ? 1.f : 0.f;
    *reinterpret_cast<float4*>(dst) = v;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    for (long e = q1 * 4; e < n1; ++e) y1[e] = (e % E1 == E1 - 1) ? 1.f : 0.f;
    for (long e = q2 * 4; e < n2; ++e) y2[e] = (e % E1 == E1 - 1) ? 1.f : 0.f;
    for (long e = q3 * 4; e < n3; ++e) y3[e] = (e % E1 == E1 - 1) ? 1.f : 0.f;
  }
}

struct PBoxParams {
  const float* boxes;      // [n, vmax, 5] x_min, y_min, x_max, y_max, mixup weight
  const int* labels;       // [n, vmax]
  const int* counts;       // [n] valid boxes per image (<= vmax)
  int n, vmax, C;
  int gw[3], gh[3];        // grid sizes of y_true_13 / _26 / _52 (named after the 416 case)
  float* y[3];
  float aw[9], ah[9];      // anchors, reference order (small -> large)
};

static constexpr int PBOX_MAX = 256;   // boxes per image handled by one CTA

// One CTA per image.  Phase 1: every box picks its best anchor (IoU of the centred sizes, first maximum wins like
// np.argmax) and its grid cell.  Phase 2: the reference writes the boxes in list order, so for a (scale, cell, anchor)
// slot hit by several boxes the LAST one's coordinates / mix weight survive while every box's class bit stays set.
__global__ void __launch_bounds__(PBOX_MAX) process_box_kernel(const PBoxParams p) {
  __shared__ int s_slot[PBOX_MAX];     // linear slot id (scale, y, x, k) or -1
  const int img = blockIdx.x;
  const int v = min(p.counts[img], p.vmax);
  const int i = threadIdx.x;
  float cx = 0.f, cy = 0.f, sw = 0.f, sh = 0.f, mixw = 0.f;
  int g = 0, k = 0, gx = 0, gy = 0, cls = 0, slot = -1;
  if (i < v) {
    const float* b = p.boxes + ((long)img * p.vmax + i) * 5;
    const float x0 = b[0], y0 = b[1], x1 = b[2], y1 = b[3];
    mixw = b[4];
    cx = __fdiv_rn(__fadd_rn(x0, x1), 2.f);          // (boxes[:, 0:2] + boxes[:, 2:4]) / 2
    cy = __fdiv_rn(__fadd_rn(y0, y1), 2.f);
    sw = __fsub_rn(x1, x0);                          // boxes[:, 2:4] - boxes[:, 0:2]
    sh = __fsub_rn(y1, y0);
    const float hw = __fdiv_rn(sw, 2.f), hh = __fdiv_rn(sh, 2.f);
    float best = 0.f;
    int bi = 0;
#pragma unroll
    for (int a = 0; a < 9; ++a) {
      const float aw2 = __fdiv_rn(p.aw[a], 2.f), ah2 = __fdiv_rn(p.ah[a], 2.f);
      const float w = __fsub_rn(fminf(hw, aw2), fmaxf(-hw, -aw2));    // maxs - mins
      const float h = __fsub_rn(fminf(hh, ah2), fmaxf(-hh, -ah2));
      const float inter = __fmul_rn(w, h);
      const float den = __fadd_rn(__fsub_rn(__fadd_rn(__fmul_rn(sw, sh), __fmul_rn(p.aw[a], p.ah[a])), inter), 1e-10f);
      const float iou = __fdiv_rn(inter, den);
      if (a == 0 || iou > best) { best = iou; bi = a; }               // np.argmax: first maximum
    }
    g = 2 - bi / 3;                                  // 0,1,2 -> y_true_52 ; 6,7,8 -> y_true_13
    k = bi % 3;
    const float ratio = g == 0 ? 32.f : (g == 1 ? 16.f : 8.f);
    gx = (int)floorf(__fdiv_rn(cx, ratio));
    gy = (int)floorf(__fdiv_rn(cy, ratio));
    cls = p.labels[(long)img * p.vmax + i];
    if (gx >= 0 && gx < p.gw[g] && gy >= 0 && gy < p.gh[g] && cls >= 0 && cls < p.C)
      slot = ((g * 4096 + gy) * 4096 + gx) * 3 + k;  // (the reference raises IndexError for a box outside the image)
  }
  s_slot[i] = slot;
  __syncthreads();
  if (slot < 0) return;
  bool last = true;
  for (int j = i + 1; j < v; ++j)
    if (s_slot[j] == slot) { last = false; break; }
  const int E1 = 6 + p.C;
  float* rec = p.y[g] + ((((long)img * p.gh[g] + gy) * p.gw[g] + gx) * 3 + k) * E1;
  rec[5 + cls] = 1.f;                                // every box leaves its class bit
  if (last) {
    rec[0] = cx; rec[1] = cy; rec[2] = sw; rec[3] = sh;
    rec[4] = 1.f;
    rec[E1 - 1] = mixw;
  }
}

// letterbox_resize(img, new_w, new_h, interp=0) -> cvtColor(BGR2RGB) -> float32 / 255
__global__ void __launch_bounds__(256)
letterbox_kernel(const uint8_t* __restrict__ src, int sh, int sw, long src_pitch, int rh, int rw, int dh, int dw, int nh,
                 int nw, double ify, double ifx, float* __restrict__ dst) {
  const long total = (long)nh * nw;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int y = (int)(i / nw), x = (int)(i - (long)y * nw);
    float r = 128.f, g = 128.f, b = 128.f;          // np.full(..., 128, np.uint8)
    const int ry = y - dh, rx = x - dw;
    if (ry >= 0 && ry < rh && rx >= 0 && rx < rw) {
      // OpenCV resizeNN: src index = min(floor(dst index * (1 / (dst size / src size))), src size - 1), in double
      const int sy = min((int)floor(ry * ify), sh - 1);
      const int sx = min((int)floor(rx * ifx), sw - 1);
      const uint8_t* px = src + (long)sy * src_pitch + (long)sx * 3;
      b = (float)px[0]; g = (float)px[1]; r = (float)px[2];
    }
    float* o = dst + i * 3;
    o[0] = __fdiv_rn(r, 255.f); o[1] = __fdiv_rn(g, 255.f); o[2] = __fdiv_rn(b, 255.f);
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// The evaluation input path for a batch of images of different sizes: parse_data(mode='val') (utils/data_utils.py:166-
// 176: resize_with_bbox(interp=1) + BGR->RGB + / 255), eval.py / eval_voc.py (stretch), test_single_image.py (stretch
// or letterbox, then the detections mapped back to the source image).
// ---------------------------------------------------------------------------------------------------------------------

static constexpr int RESIZE_MAX_SIDE = 1 << 20;      // source image sides; keeps every index product in int32

// letterbox_resize's scalars (utils/data_aug.py:279-289); stretch is the whole target with no border.  Host and device
// share this so the box kernels see exactly the geometry the host validated.
struct ResizeGeom {
  double ratio;        // letterbox resize_ratio
  int rh, rw, dh, dw;  // resized size and border offsets
};
__host__ __device__ inline ResizeGeom resize_geom(int sh, int sw, int nh, int nw, int letterbox) {
  ResizeGeom g;
  if (letterbox) {
    const double a = (double)nw / (double)sw, b = (double)nh / (double)sh;
    g.ratio = a < b ? a : b;
    g.rw = (int)(g.ratio * sw);
    g.rh = (int)(g.ratio * sh);
    g.dw = (int)((nw - g.rw) / 2.0);
    g.dh = (int)((nh - g.rh) / 2.0);
  } else {
    g.ratio = 0.0; g.rh = nh; g.rw = nw; g.dh = 0; g.dw = 0;
  }
  return g;
}

// OpenCV's linear source coordinate: f = (float)((d + 0.5) * scale - 0.5), s = floor(f), f -= s (resize.cpp,
// resizeGeneric setup).  Double ops spelled _rn so no FMA is contracted.
struct LinTap { int s; float f; };
__device__ __forceinline__ LinTap linear_tap(int d, double scale) {
  float f = __double2float_rn(__dsub_rn(__dmul_rn((double)d + 0.5, scale), 0.5));
  const int s = (int)floorf(f);
  f = __fsub_rn(f, (float)s);
  return {s, f};
}
// saturate_cast<short>(w * INTER_RESIZE_COEF_SCALE): round half to even
__device__ __forceinline__ int coef11(float w) { return __float2int_rn(__fmul_rn(w, 2048.f)); }

struct ImgDesc { long off; int h, w; long pitch; };   // one row of the int64 [n, 4] descriptor table

// ---------------------------------------------------------------------------------------------------------------------
// Per-image interpolation tables of cv2.resize's other modes (INTER_CUBIC, INTER_AREA, INTER_LANCZOS4), built on the
// host as OpenCV builds them (resize.cpp: resize(), computeResizeAreaTab) and sent in one buffer:
//   ResizeTab[n] headers, then per image (16-byte aligned) its x table and y table.
// ---------------------------------------------------------------------------------------------------------------------
enum ResizeMode : int {
  RM_NEAREST = 0, RM_LINEAR = 1,       // computed on the device, as yb_resize_batch
  RM_CUBIC = 2, RM_LANCZOS4 = 4,       // GenTap tables, 4 / 8 taps
  RM_COPY = 5,                         // same size in and out: cv2.resize copies
  RM_AREA_FAST = 6,                    // both axes shrink by integers: block mean over kx x ky
  RM_AREA_FLOAT = 7,                   // both axes shrink: AreaSpan + AreaTap runs, float32 sums
  RM_AREA_LINEAR = 8,                  // an axis grows: bilinear with area-mode coefficients (GenTap, 2 taps)
};
struct ResizeTab {                     // 64 bytes
  int interp, mode;
  int src_h, src_w, rh, rw;            // what the table was built for, checked against the call
  int kx, ky;                          // RM_AREA_FAST block
  long long x_off, y_off;              // byte offsets (in the whole buffer) of the GenTap / AreaSpan arrays
  long long xt_off, yt_off;            // RM_AREA_FLOAT: byte offsets of the AreaTap runs
};
struct GenTap { int s; short c[8]; };  // first source index (unclamped; RM_AREA_LINEAR: clamped) and int16 coefficients
struct AreaSpan { int start, count; }; // a destination index's run in the AreaTap list
struct AreaTap { int s; float a; };    // computeResizeAreaTab's (source index, alpha)

// ---- the per-pixel paths: one output pixel's B, G, R (uint8 values) --------------------------------------------------

// resizeNN, as letterbox_kernel
__device__ __forceinline__ void px_nearest(const uint8_t* im, const ImgDesc& d, int rx, int ry, double scx, double scy,
                                           int v[3]) {
  const int sy = min((int)floor(ry * scy), d.h - 1);
  const int sx = min((int)floor(rx * scx), d.w - 1);
  const uint8_t* px = im + (long)sy * d.pitch + sx * 3;
  v[0] = px[0]; v[1] = px[1]; v[2] = px[2];
}

// OpenCV's fixed-point bilinear: x taps sx (clamped) and min(sx + 1, w - 1) with cx0 / cx1, rows sy and sy + 1 clamped
// with cy0 / cy1.
__device__ __forceinline__ void px_bilinear(const uint8_t* im, const ImgDesc& d, int sx, int cx0, int cx1, int sy,
                                            int cy0, int cy1, int v[3]) {
  const int x0 = sx * 3, x1 = min(sx + 1, d.w - 1) * 3;
  const uint8_t* r0 = im + (long)min(max(sy, 0), d.h - 1) * d.pitch;
  const uint8_t* r1 = im + (long)min(max(sy + 1, 0), d.h - 1) * d.pitch;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const int h0 = r0[x0 + c] * cx0 + r0[x1 + c] * cx1;          // horizontal pass, int32
    const int h1 = r1[x0 + c] * cx0 + r1[x1 + c] * cx1;
    // vertical pass as OpenCV's SIMD VResizeLinearVec_32s8u: (h >> 4) * c as int16 mul_hi, +2 >> 2, saturate
    const int t = (((h0 >> 4) * cy0) >> 16) + (((h1 >> 4) * cy1) >> 16);
    v[c] = min(max((t + 2) >> 2, 0), 255);
  }
}

// INTER_LINEAR: the taps from linear_tap.  x: a source column outside [0, w - 1) takes that border pixel with weight 1
// (fraction zeroed); y: the fraction is kept, only the two row indices are clamped.
__device__ __forceinline__ void px_linear(const uint8_t* im, const ImgDesc& d, int rx, int ry, double scx, double scy,
                                          int v[3]) {
  LinTap tx = linear_tap(rx, scx);
  if (tx.s < 0) { tx.s = 0; tx.f = 0.f; }
  if (tx.s >= d.w - 1) { tx.s = d.w - 1; tx.f = 0.f; }
  const LinTap ty = linear_tap(ry, scy);
  px_bilinear(im, d, tx.s, coef11(__fsub_rn(1.f, tx.f)), coef11(tx.f), ty.s, coef11(__fsub_rn(1.f, ty.f)),
              coef11(ty.f), v);
}

// INTER_CUBIC (K = 4) / INTER_LANCZOS4 (K = 8), resizeGeneric_ with border-replicated taps: an int32 horizontal pass
// per source row, then the vertical pass.  Lanczos4's is VResizeLanczos4: int32, (sum + 2^21) >> 22.  Cubic's is
// VResizeCubicVec_32s8u on a row's first nvec = 8 * floor(3 rw / 8) values (float32: h * (beta * 2^-22), summed from
// the last row outwards, rounded half to even) and the scalar int32 form on the rest; e0 = 3 * rx is the pixel's first
// value in its row.
template <int K>
__device__ __forceinline__ void px_generic(const uint8_t* im, const ImgDesc& d, const GenTap& tx, const GenTap& ty,
                                           int e0, int nvec, int v[3]) {
  int xo[K];
#pragma unroll
  for (int j = 0; j < K; ++j) xo[j] = min(max(tx.s + j, 0), d.w - 1) * 3;
  int hs[K][3];
#pragma unroll
  for (int k = 0; k < K; ++k) {
    const uint8_t* row = im + (long)min(max(ty.s + k, 0), d.h - 1) * d.pitch;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      int h = 0;
#pragma unroll
      for (int j = 0; j < K; ++j) h += row[xo[j] + c] * (int)tx.c[j];
      hs[k][c] = h;
    }
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    int r;
    if (K == 4 && e0 + c < nvec) {
      const float sc = 1.f / (2048.f * 2048.f);
      float acc = __fmul_rn((float)hs[3][c], __fmul_rn((float)ty.c[3], sc));
      acc = __fadd_rn(__fmul_rn((float)hs[2][c], __fmul_rn((float)ty.c[2], sc)), acc);
      acc = __fadd_rn(__fmul_rn((float)hs[1][c], __fmul_rn((float)ty.c[1], sc)), acc);
      acc = __fadd_rn(__fmul_rn((float)hs[0][c], __fmul_rn((float)ty.c[0], sc)), acc);
      r = __float2int_rn(acc);
    } else {
      int s = 0;
#pragma unroll
      for (int k = 0; k < K; ++k) s += hs[k][c] * (int)ty.c[k];
      r = (s + (1 << 21)) >> 22;
    }
    v[c] = min(max(r, 0), 255);
  }
}

// INTER_AREA, integer shrink on both axes (ResizeAreaFast): the kx x ky block sum; 2 x 2 rounds (s + 2) >> 2 as
// OpenCV's ResizeAreaFastVec, every other block rint(s * (1.f / area)).
__device__ __forceinline__ void px_area_fast(const uint8_t* im, const ImgDesc& d, int rx, int ry, int kx, int ky,
                                             int v[3]) {
  int s[3] = {0, 0, 0};
  for (int yy = 0; yy < ky; ++yy) {
    const uint8_t* row = im + (long)(ry * ky + yy) * d.pitch + (long)rx * kx * 3;
    for (int xx = 0; xx < kx * 3; xx += 3) {
      s[0] += row[xx]; s[1] += row[xx + 1]; s[2] += row[xx + 2];
    }
  }
  const float scale = __fdiv_rn(1.f, (float)(kx * ky));
#pragma unroll
  for (int c = 0; c < 3; ++c)
    v[c] = (kx == 2 && ky == 2) ? (s[c] + 2) >> 2 : min(max(__float2int_rn(__fmul_rn((float)s[c], scale)), 0), 255);
}

// INTER_AREA, both axes shrinking (ResizeArea_Invoker): per source row of the y run buf = sum S * alpha over the x run,
// then sum = sum beta * buf, float32 in table order; saturate_cast<uchar> rounds half to even.
__device__ __forceinline__ void px_area_float(const uint8_t* im, const ImgDesc& d, const AreaSpan& sx,
                                              const AreaSpan& sy, const AreaTap* __restrict__ xt,
                                              const AreaTap* __restrict__ yt, int v[3]) {
  float acc[3] = {0.f, 0.f, 0.f};
  for (int j = 0; j < sy.count; ++j) {
    const AreaTap ty = yt[sy.start + j];
    const uint8_t* row = im + (long)ty.s * d.pitch;
    float buf[3] = {0.f, 0.f, 0.f};
    for (int i = 0; i < sx.count; ++i) {
      const AreaTap tx = xt[sx.start + i];
      const uint8_t* p = row + tx.s * 3;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float m = __fmul_rn((float)p[c], tx.a);
        buf[c] = i == 0 ? m : __fadd_rn(buf[c], m);
      }
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float m = __fmul_rn(ty.a, buf[c]);
      acc[c] = j == 0 ? m : __fadd_rn(acc[c], m);
    }
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) v[c] = min(max(__float2int_rn(acc[c]), 0), 255);
}

// grid (blocks per image, n): block (bx, img) covers pixels bx, bx + gridDim.x, ... (x 256) of output image img.
// letterbox_resize / cv2.resize(interp) -> cvtColor(BGR2RGB) -> float32 / 255.  tabs == nullptr: every image takes
// `interp` (0 or 1); otherwise each image takes its ResizeTab's mode.  TABS = false compiles only the first two paths.
template <bool TABS>
__global__ void __launch_bounds__(256)
resize_batch_kernel(const uint8_t* __restrict__ src, const int64_t* __restrict__ desc, int nh, int nw, int letterbox,
                    int interp, const uint8_t* __restrict__ tabs, float* __restrict__ dst,
                    double* __restrict__ params) {
  __shared__ ImgDesc s_d;
  __shared__ ResizeGeom s_g;
  __shared__ ResizeTab s_t;
  const int img = blockIdx.y;
  if (threadIdx.x == 0) {
    const int64_t* d = desc + 4L * img;
    s_d = {(long)d[0], (int)d[1], (int)d[2], (long)d[3]};
    s_g = resize_geom(s_d.h, s_d.w, nh, nw, letterbox);
    if (TABS) s_t = reinterpret_cast<const ResizeTab*>(tabs)[img];
    else s_t.mode = interp;
    if (params && blockIdx.x == 0) {
      double* p = params + 4L * img;
      if (letterbox) { p[0] = s_g.ratio; p[1] = s_g.dw; p[2] = s_g.dh; p[3] = 1.0; }
      else { p[0] = (double)s_d.w / (double)nw; p[1] = (double)s_d.h / (double)nh; p[2] = 0.0; p[3] = 0.0; }
    }
  }
  __syncthreads();
  const ImgDesc d = s_d;
  const ResizeGeom g = s_g;
  const ResizeTab t = s_t;
  const uint8_t* im = src + d.off;
  // OpenCV: inv_scale = dsize / ssize; scale = 1. / inv_scale (resizeNN's ifx / resizeGeneric's scale_x alike)
  const double scx = 1.0 / ((double)g.rw / (double)d.w), scy = 1.0 / ((double)g.rh / (double)d.h);
  const int nvec = g.rw * 3 / 8 * 8;
  const long total = (long)nh * nw;
  float* out = dst + (long)img * total * 3;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int y = (int)(i / nw), x = (int)(i - (long)y * nw);
    int v[3] = {128, 128, 128};                     // np.full(..., 128, np.uint8)
    const int ry = y - g.dh, rx = x - g.dw;
    if (ry >= 0 && ry < g.rh && rx >= 0 && rx < g.rw) {
      if (!TABS) {
        if (t.mode == RM_NEAREST) px_nearest(im, d, rx, ry, scx, scy, v);
        else px_linear(im, d, rx, ry, scx, scy, v);
      } else switch (t.mode) {
        case RM_NEAREST: px_nearest(im, d, rx, ry, scx, scy, v); break;
        case RM_LINEAR: px_linear(im, d, rx, ry, scx, scy, v); break;
        case RM_COPY: {
          const uint8_t* px = im + (long)ry * d.pitch + rx * 3;
          v[0] = px[0]; v[1] = px[1]; v[2] = px[2];
          break;
        }
        case RM_CUBIC:
        case RM_LANCZOS4: {
          const GenTap tx = reinterpret_cast<const GenTap*>(tabs + t.x_off)[rx];
          const GenTap ty = reinterpret_cast<const GenTap*>(tabs + t.y_off)[ry];
          if (t.mode == RM_CUBIC) px_generic<4>(im, d, tx, ty, rx * 3, nvec, v);
          else px_generic<8>(im, d, tx, ty, rx * 3, nvec, v);
          break;
        }
        case RM_AREA_FAST: px_area_fast(im, d, rx, ry, t.kx, t.ky, v); break;
        case RM_AREA_FLOAT:
          px_area_float(im, d, reinterpret_cast<const AreaSpan*>(tabs + t.x_off)[rx],
                        reinterpret_cast<const AreaSpan*>(tabs + t.y_off)[ry],
                        reinterpret_cast<const AreaTap*>(tabs + t.xt_off), reinterpret_cast<const AreaTap*>(tabs + t.yt_off),
                        v);
          break;
        default: {                                  // RM_AREA_LINEAR
          const GenTap tx = reinterpret_cast<const GenTap*>(tabs + t.x_off)[rx];
          const GenTap ty = reinterpret_cast<const GenTap*>(tabs + t.y_off)[ry];
          px_bilinear(im, d, tx.s, tx.c[0], tx.c[1], ty.s, ty.c[0], ty.c[1], v);
        }
      }
    }
    float* o = out + i * 3;
    o[0] = __fdiv_rn((float)v[2], 255.f); o[1] = __fdiv_rn((float)v[1], 255.f); o[2] = __fdiv_rn((float)v[0], 255.f);
  }
}

// resize_with_bbox's box lines (utils/data_aug.py:301-318) in place, float32 in the reference's order; the Python
// float / int scalars act as float32 under numpy 2 (NEP 50).  One thread per box slot.
__global__ void __launch_bounds__(256)
resize_boxes_kernel(float* __restrict__ boxes, const int32_t* __restrict__ counts, int n, int vmax, int ld,
                    const int64_t* __restrict__ desc, int nh, int nw, int letterbox) {
  const long t = blockIdx.x * (long)blockDim.x + threadIdx.x;
  if (t >= (long)n * vmax) return;
  const int img = (int)(t / vmax), j = (int)(t - (long)img * vmax);
  if (j >= min(counts[img], vmax)) return;
  const int sh = (int)desc[4L * img + 1], sw = (int)desc[4L * img + 2];
  float* b = boxes + t * ld;
  if (letterbox) {                                  // bbox * resize_ratio + dw / dh
    const ResizeGeom g = resize_geom(sh, sw, nh, nw, 1);
    const float r = __double2float_rn(g.ratio), dw = (float)g.dw, dh = (float)g.dh;
    b[0] = __fadd_rn(__fmul_rn(b[0], r), dw); b[2] = __fadd_rn(__fmul_rn(b[2], r), dw);
    b[1] = __fadd_rn(__fmul_rn(b[1], r), dh); b[3] = __fadd_rn(__fmul_rn(b[3], r), dh);
  } else {                                          // bbox / ori_width * new_width
    const float fw = (float)sw, fh = (float)sh, fnw = (float)nw, fnh = (float)nh;
    b[0] = __fmul_rn(__fdiv_rn(b[0], fw), fnw); b[2] = __fmul_rn(__fdiv_rn(b[2], fw), fnw);
    b[1] = __fmul_rn(__fdiv_rn(b[1], fh), fnh); b[3] = __fmul_rn(__fdiv_rn(b[3], fh), fnh);
  }
}

// test_single_image.py:64-70 in place: letterbox (b - dw) / resize_ratio, stretch b * (ori / new), float32.
__global__ void __launch_bounds__(256)
restore_boxes_kernel(float* __restrict__ boxes, const int32_t* __restrict__ counts, int n, int slots, int ld,
                     const double* __restrict__ params) {
  const long t = blockIdx.x * (long)blockDim.x + threadIdx.x;
  if (t >= (long)n * slots) return;
  const int img = (int)(t / slots), j = (int)(t - (long)img * slots);
  if (j >= min(counts[img], slots)) return;
  const double* p = params + 4L * img;
  float* b = boxes + t * ld;
  if (p[3] != 0.0) {
    const float r = __double2float_rn(p[0]), dw = __double2float_rn(p[1]), dh = __double2float_rn(p[2]);
    b[0] = __fdiv_rn(__fsub_rn(b[0], dw), r); b[2] = __fdiv_rn(__fsub_rn(b[2], dw), r);
    b[1] = __fdiv_rn(__fsub_rn(b[1], dh), r); b[3] = __fdiv_rn(__fsub_rn(b[3], dh), r);
  } else {
    const float fx = __double2float_rn(p[0]), fy = __double2float_rn(p[1]);
    b[0] = __fmul_rn(b[0], fx); b[2] = __fmul_rn(b[2], fx);
    b[1] = __fmul_rn(b[1], fy); b[3] = __fmul_rn(b[3], fy);
  }
}

// ---- host: the tables, as OpenCV's resize() and computeResizeAreaTab build them (plain C++: glibc's sin / cos) ------

// interpolateCubic, float32, A = -0.75
static void cubic_coeffs(float x, float* c) {
  const float A = -0.75f;
  c[0] = ((A * (x + 1) - 5 * A) * (x + 1) + 8 * A) * (x + 1) - 4 * A;
  c[1] = ((A + 2) * x - (A + 3)) * x * x + 1;
  c[2] = ((A + 2) * (1 - x) - (A + 3)) * (1 - x) * (1 - x) + 1;
  c[3] = 1.f - c[0] - c[1] - c[2];
}

// interpolateLanczos4: double sin / cos, float32 coefficients normalised by the reciprocal of their float32 sum
static void lanczos4_coeffs(float x, float* c) {
  static const double s45 = 0.70710678118654752440084436210485;
  static const double cs[8][2] = {{1, 0}, {-s45, -s45}, {0, 1}, {s45, -s45}, {-1, 0}, {s45, s45}, {0, -1}, {-s45, s45}};
  const double pi = 3.1415926535897932384626433832795;
  float sum = 0;
  const double y0 = -(x + 3) * pi * 0.25, s0 = std::sin(y0), c0 = std::cos(y0);
  for (int i = 0; i < 8; ++i) {
    const float yi = x + 3 - i;
    if (std::fabs(yi) >= 1e-6f) {
      const double y = -yi * pi * 0.25;
      c[i] = (float)((cs[i][0] * s0 + cs[i][1] * c0) / (y * y));
    } else {
      c[i] = 1e30f;                                  // x ~ 0: the coefficients become 0 0 0 1 0 0 0 0
    }
    sum += c[i];
  }
  sum = 1.f / sum;
  for (int i = 0; i < 8; ++i) c[i] *= sum;
}

static short coef11_host(float c) {                  // saturate_cast<short>(c * INTER_RESIZE_COEF_SCALE)
  const long v = std::lrint(c * 2048.f);
  return (short)(v < -32768 ? -32768 : (v > 32767 ? 32767 : v));
}

// resize()'s per-axis setup for cubic / Lanczos4 (generic source coordinate) or area-as-linear (area coordinate);
// clamp_x applies the x axis's border rule of the 2-tap path (a source past the last column takes it with weight 1).
static void gen_table(int dsize, int ssize, int interp, bool clamp_x, GenTap* tab) {
  const double inv = (double)dsize / (double)ssize, scale = 1.0 / inv;
  const int ksize = interp == RM_CUBIC ? 4 : interp == RM_LANCZOS4 ? 8 : 2;
  for (int d = 0; d < dsize; ++d) {
    int s;
    float f;
    if (ksize != 2) {
      f = (float)((d + 0.5) * scale - 0.5);
      s = (int)std::floor(f);
      f -= s;
    } else {
      s = (int)std::floor(d * scale);
      f = (float)((d + 1) - (s + 1) * inv);
      f = f <= 0 ? 0.f : f - (float)std::floor(f);
      if (clamp_x && s >= ssize - 1) { f = 0.f; s = ssize - 1; }
    }
    float cbuf[8] = {0.f};
    if (ksize == 4) cubic_coeffs(f, cbuf);
    else if (ksize == 8) lanczos4_coeffs(f, cbuf);
    else { cbuf[0] = 1.f - f; cbuf[1] = f; }
    GenTap t;
    std::memset(&t, 0, sizeof(t));
    t.s = ksize == 2 ? s : s - ksize / 2 + 1;
    for (int k = 0; k < ksize; ++k) t.c[k] = coef11_host(cbuf[k]);
    tab[d] = t;
  }
}

// computeResizeAreaTab: spans (if not null) and taps (if not null) of one axis; returns the number of taps
static int area_table(int ssize, int dsize, AreaSpan* spans, AreaTap* taps) {
  const double scale = 1.0 / ((double)dsize / (double)ssize);
  int k = 0;
  for (int dx = 0; dx < dsize; ++dx) {
    const double fsx1 = dx * scale, fsx2 = fsx1 + scale;
    const double cell = std::min(scale, ssize - fsx1);
    int sx1 = (int)std::ceil(fsx1), sx2 = (int)std::floor(fsx2);
    sx2 = std::min(sx2, ssize - 1);
    sx1 = std::min(sx1, sx2);
    const int k0 = k;
    if (sx1 - fsx1 > 1e-3) {
      if (taps) taps[k] = {sx1 - 1, (float)((sx1 - fsx1) / cell)};
      ++k;
    }
    for (int sx = sx1; sx < sx2; ++sx) {
      if (taps) taps[k] = {sx, (float)(1.0 / cell)};
      ++k;
    }
    if (fsx2 - sx2 > 1e-3) {
      if (taps) taps[k] = {sx2, (float)(std::min(std::min(fsx2 - sx2, 1.), cell) / cell)};
      ++k;
    }
    if (spans) spans[dx] = {k0, k - k0};
  }
  return k;
}

// resize()'s choice for a uint8 image of (sh, sw) -> (rh, rw) at OpenCV interpolation `interp` (0..4)
static int resize_mode(int interp, int sh, int sw, int rh, int rw, int* kx, int* ky) {
  *kx = *ky = 0;
  if (interp <= 1) return interp;
  if (sh == rh && sw == rw) return RM_COPY;
  if (interp != 3) return interp;
  const double scx = 1.0 / ((double)rw / (double)sw), scy = 1.0 / ((double)rh / (double)sh);
  const int ix = (int)std::lrint(scx), iy = (int)std::lrint(scy);
  if (scx >= 1 && scy >= 1) {
    if (std::fabs(scx - ix) < DBL_EPSILON && std::fabs(scy - iy) < DBL_EPSILON) {
      *kx = ix; *ky = iy;
      return RM_AREA_FAST;
    }
    return RM_AREA_FLOAT;
  }
  return RM_AREA_LINEAR;
}

static inline size_t align16(size_t v) { return (v + 15) & ~(size_t)15; }

// Lays out (and with `out` fills) the whole table buffer; returns its size.
static size_t resize_tables_build(const int64_t* desc, int n, int nh, int nw, int letterbox, const int32_t* interp,
                                  uint8_t* out) {
  size_t off = align16(sizeof(ResizeTab) * (size_t)n);
  for (int i = 0; i < n; ++i) {
    const int sh = (int)desc[4L * i + 1], sw = (int)desc[4L * i + 2];
    const ResizeGeom g = resize_geom(sh, sw, nh, nw, letterbox);
    ResizeTab t;
    std::memset(&t, 0, sizeof(t));
    t.interp = interp[i];
    t.src_h = sh; t.src_w = sw; t.rh = g.rh; t.rw = g.rw;
    t.mode = resize_mode(interp[i], sh, sw, g.rh, g.rw, &t.kx, &t.ky);
    if (t.mode == RM_CUBIC || t.mode == RM_LANCZOS4 || t.mode == RM_AREA_LINEAR) {
      t.x_off = (long long)off;
      off = align16(off + sizeof(GenTap) * (size_t)g.rw);
      t.y_off = (long long)off;
      off = align16(off + sizeof(GenTap) * (size_t)g.rh);
      if (out) {
        gen_table(g.rw, sw, t.mode, true, reinterpret_cast<GenTap*>(out + t.x_off));
        gen_table(g.rh, sh, t.mode, false, reinterpret_cast<GenTap*>(out + t.y_off));
      }
    } else if (t.mode == RM_AREA_FLOAT) {
      const size_t nx = (size_t)area_table(sw, g.rw, nullptr, nullptr), ny = (size_t)area_table(sh, g.rh, nullptr, nullptr);
      t.x_off = (long long)off; off = align16(off + sizeof(AreaSpan) * (size_t)g.rw);
      t.y_off = (long long)off; off = align16(off + sizeof(AreaSpan) * (size_t)g.rh);
      t.xt_off = (long long)off; off = align16(off + sizeof(AreaTap) * nx);
      t.yt_off = (long long)off; off = align16(off + sizeof(AreaTap) * ny);
      if (out) {
        area_table(sw, g.rw, reinterpret_cast<AreaSpan*>(out + t.x_off), reinterpret_cast<AreaTap*>(out + t.xt_off));
        area_table(sh, g.rh, reinterpret_cast<AreaSpan*>(out + t.y_off), reinterpret_cast<AreaTap*>(out + t.yt_off));
      }
    }
    if (out) std::memcpy(out + sizeof(ResizeTab) * (size_t)i, &t, sizeof(t));
  }
  return off;
}

// Everything yb_resize_batch checks, plus the interpolations 0..4; device pointers are not touched.
static int resize_interp_check(const int64_t* desc_host, long images_bytes, int n, int new_h, int new_w, int letterbox,
                               const int32_t* interp_host, const char* what) {
  YB_REQUIRE(desc_host && interp_host, "%s: null host pointer", what);
  YB_REQUIRE(n > 0 && n <= 65535, "%s: n must be in 1..65535 (got %d)", what, n);
  YB_REQUIRE(new_h > 0 && new_w > 0, "%s: target size must be positive (got %dx%d)", what, new_w, new_h);
  YB_REQUIRE(letterbox == 0 || letterbox == 1, "%s: letterbox must be 0 or 1 (got %d)", what, letterbox);
  for (int i = 0; i < n; ++i) {
    YB_REQUIRE(interp_host[i] >= 0 && interp_host[i] <= 4,
               "%s: image %d: interp must be 0 (nearest), 1 (linear), 2 (cubic), 3 (area) or 4 (Lanczos4), got %d", what,
               i, interp_host[i]);
    const int64_t off = desc_host[4L * i], h = desc_host[4L * i + 1], w = desc_host[4L * i + 2], pitch = desc_host[4L * i + 3];
    YB_REQUIRE(h > 0 && w > 0 && h <= RESIZE_MAX_SIDE && w <= RESIZE_MAX_SIDE, "%s: image %d has size %lldx%lld", what, i,
               (long long)w, (long long)h);
    YB_REQUIRE(images_bytes < 0 || (off >= 0 && pitch >= 3 * w && off + (h - 1) * pitch + 3 * w <= images_bytes),
               "%s: image %d (offset %lld, pitch %lld) lies outside the %ld-byte buffer", what, i, (long long)off,
               (long long)pitch, images_bytes);
    const ResizeGeom g = resize_geom((int)h, (int)w, new_h, new_w, letterbox);
    YB_REQUIRE(g.rh > 0 && g.rw > 0, "%s: image %d (%lldx%lld) letterboxes to an empty resize", what, i, (long long)w,
               (long long)h);
  }
  return YB_OK;
}

}  // namespace yb

using namespace yb;

extern "C" int yb_process_box(const float* boxes, const int32_t* labels, const int32_t* counts, int n, int vmax,
                              int img_w, int img_h, int class_num, const float* anchors9x2, float* y_true_1,
                              float* y_true_2, float* y_true_3, void* stream) {
  YB_REQUIRE(boxes && labels && counts && anchors9x2 && y_true_1 && y_true_2 && y_true_3, "process_box: null pointer");
  YB_REQUIRE(n > 0 && vmax > 0 && vmax <= PBOX_MAX, "process_box: vmax must be in 1..%d (got %d)", PBOX_MAX, vmax);
  YB_REQUIRE(class_num > 0 && img_w > 0 && img_h > 0 && img_w % 32 == 0 && img_h % 32 == 0 && img_w / 8 < 4096 && img_h / 8 < 4096,
             "process_box: image size must be a multiple of 32 (got %dx%d)", img_w, img_h);
  YB_REQUIRE(((uintptr_t)y_true_1 & 15) == 0 && ((uintptr_t)y_true_2 & 15) == 0 && ((uintptr_t)y_true_3 & 15) == 0,
             "process_box: y_true tensors must be 16-byte aligned");
  PBoxParams p;
  p.boxes = boxes; p.labels = labels; p.counts = counts; p.n = n; p.vmax = vmax; p.C = class_num;
  const int div[3] = {32, 16, 8};
  long cnt[3];
  float* ys[3] = {y_true_1, y_true_2, y_true_3};
  for (int s = 0; s < 3; ++s) {
    p.gw[s] = img_w / div[s]; p.gh[s] = img_h / div[s]; p.y[s] = ys[s];
    cnt[s] = (long)n * p.gh[s] * p.gw[s] * 3 * (6 + class_num);
  }
  for (int a = 0; a < 9; ++a) { p.aw[a] = anchors9x2[2 * a]; p.ah[a] = anchors9x2[2 * a + 1]; }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long total4 = (cnt[0] + cnt[1] + cnt[2]) / 4;
  long blocks = (total4 + 255) / 256;
  const long cap = (long)num_sms() * 16;
  if (blocks > cap) blocks = cap;
  ytrue_fill_kernel<<<(int)blocks, 256, 0, st>>>(y_true_1, cnt[0], y_true_2, cnt[1], y_true_3, cnt[2], 6 + class_num);
  YB_CUDA(cudaGetLastError());
  process_box_kernel<<<n, PBOX_MAX, 0, st>>>(p);
  YB_CUDA(cudaGetLastError());
  return YB_OK;
}

extern "C" int yb_letterbox_params(int src_h, int src_w, int new_h, int new_w, double* resize_ratio, int* resize_h,
                                   int* resize_w, int* dh, int* dw) {
  YB_REQUIRE(src_h > 0 && src_w > 0 && new_h > 0 && new_w > 0 && resize_ratio && resize_h && resize_w && dh && dw,
             "letterbox_params: bad argument");
  const double a = (double)new_w / (double)src_w, b = (double)new_h / (double)src_h;    // utils/data_aug.py:280
  const double ratio = a < b ? a : b;
  *resize_ratio = ratio;
  *resize_w = (int)(ratio * src_w);                    // int(): truncation towards zero
  *resize_h = (int)(ratio * src_h);
  *dw = (int)((new_w - *resize_w) / 2.0);
  *dh = (int)((new_h - *resize_h) / 2.0);
  return YB_OK;
}

extern "C" int yb_letterbox_normalize(const uint8_t* bgr, int src_h, int src_w, long src_pitch_bytes, int new_h,
                                      int new_w, float* out_rgb, void* stream) {
  YB_REQUIRE(bgr && out_rgb && src_pitch_bytes >= 3L * src_w, "letterbox: bad argument");
  double ratio;
  int rh, rw, dh, dw;
  int rc = yb_letterbox_params(src_h, src_w, new_h, new_w, &ratio, &rh, &rw, &dh, &dw);
  if (rc) return rc;
  YB_REQUIRE(rh > 0 && rw > 0, "letterbox: image too small for the target size");
  // OpenCV: inv_scale = dsize / ssize; ifx = 1. / inv_scale  (modules/imgproc/src/resize.cpp, resizeNN)
  const double ifx = 1.0 / ((double)rw / (double)src_w), ify = 1.0 / ((double)rh / (double)src_h);
  const long total = (long)new_h * new_w;
  long blocks = (total + 255) / 256;
  const long cap = (long)num_sms() * 16;
  if (blocks > cap) blocks = cap;
  letterbox_kernel<<<(int)blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(bgr, src_h, src_w, src_pitch_bytes, rh, rw, dh,
                                                                             dw, new_h, new_w, ify, ifx, out_rgb);
  YB_CUDA(cudaGetLastError());
  return YB_OK;
}

extern "C" int yb_resize_batch(const uint8_t* images, long images_bytes, const int64_t* desc_host,
                               const int64_t* desc_dev, int n, int new_h, int new_w, int letterbox, int interp,
                               float* out_rgb, double* params, void* stream) {
  YB_REQUIRE(images && desc_host && desc_dev && out_rgb, "resize_batch: null pointer");
  YB_REQUIRE(((uintptr_t)desc_dev & 7) == 0 && ((uintptr_t)params & 7) == 0,
             "resize_batch: the descriptor table and params must be 8-byte aligned");
  YB_REQUIRE(n > 0 && n <= 65535, "resize_batch: n must be in 1..65535 (got %d)", n);
  YB_REQUIRE(new_h > 0 && new_w > 0, "resize_batch: target size must be positive (got %dx%d)", new_w, new_h);
  YB_REQUIRE(letterbox == 0 || letterbox == 1, "resize_batch: letterbox must be 0 or 1 (got %d)", letterbox);
  YB_REQUIRE(interp == 0 || interp == 1, "resize_batch: interp must be 0 (nearest) or 1 (linear), got %d", interp);
  for (int i = 0; i < n; ++i) {
    const int64_t off = desc_host[4L * i], h = desc_host[4L * i + 1], w = desc_host[4L * i + 2], pitch = desc_host[4L * i + 3];
    YB_REQUIRE(h > 0 && w > 0 && h <= RESIZE_MAX_SIDE && w <= RESIZE_MAX_SIDE,
               "resize_batch: image %d has size %lldx%lld", i, (long long)w, (long long)h);
    YB_REQUIRE(off >= 0 && pitch >= 3 * w && off + (h - 1) * pitch + 3 * w <= images_bytes,
               "resize_batch: image %d (offset %lld, pitch %lld) lies outside the %ld-byte buffer", i, (long long)off,
               (long long)pitch, images_bytes);
    const ResizeGeom g = resize_geom((int)h, (int)w, new_h, new_w, letterbox);
    YB_REQUIRE(g.rh > 0 && g.rw > 0, "resize_batch: image %d (%lldx%lld) letterboxes to an empty resize", i,
               (long long)w, (long long)h);
  }
  const long total = (long)new_h * new_w;
  long bx = (total + 255) / 256;
  const long cap = ((long)num_sms() * 16 + n - 1) / n;  // about 16 CTAs per SM over the batch, then grid-stride
  if (bx > cap) bx = cap;
  resize_batch_kernel<false><<<dim3((unsigned)bx, (unsigned)n), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      images, desc_dev, new_h, new_w, letterbox, interp, nullptr, out_rgb, params);
  YB_CUDA(cudaGetLastError());
  return YB_OK;
}

extern "C" int yb_resize_tables_bytes(const int64_t* desc_host, int n, int new_h, int new_w, int letterbox,
                                      const int32_t* interp_host, size_t* bytes) {
  YB_REQUIRE(bytes, "resize_tables_bytes: null pointer");
  const int rc = resize_interp_check(desc_host, -1, n, new_h, new_w, letterbox, interp_host, "resize_tables_bytes");
  if (rc) return rc;
  *bytes = resize_tables_build(desc_host, n, new_h, new_w, letterbox, interp_host, nullptr);
  return YB_OK;
}

extern "C" int yb_resize_tables(const int64_t* desc_host, int n, int new_h, int new_w, int letterbox,
                                const int32_t* interp_host, void* tables_host, size_t bytes) {
  YB_REQUIRE(tables_host, "resize_tables: null pointer");
  YB_REQUIRE(((uintptr_t)tables_host & 15) == 0, "resize_tables: the table buffer must be 16-byte aligned");
  const int rc = resize_interp_check(desc_host, -1, n, new_h, new_w, letterbox, interp_host, "resize_tables");
  if (rc) return rc;
  const size_t need = resize_tables_build(desc_host, n, new_h, new_w, letterbox, interp_host, nullptr);
  YB_REQUIRE(bytes == need, "resize_tables: the buffer holds %zu bytes, the tables take %zu", bytes, need);
  std::memset(tables_host, 0, bytes);
  resize_tables_build(desc_host, n, new_h, new_w, letterbox, interp_host, static_cast<uint8_t*>(tables_host));
  return YB_OK;
}

extern "C" int yb_resize_batch_interp(const uint8_t* images, long images_bytes, const int64_t* desc_host,
                                      const int64_t* desc_dev, int n, int new_h, int new_w, int letterbox,
                                      const int32_t* interp_host, const void* tables_host, const void* tables_dev,
                                      size_t tables_bytes, float* out_rgb, double* params, void* stream) {
  YB_REQUIRE(images && desc_dev && out_rgb, "resize_batch_interp: null pointer");
  YB_REQUIRE(tables_host && tables_dev, "resize_batch_interp: tables_host and tables_dev must both be given");
  YB_REQUIRE(((uintptr_t)desc_dev & 7) == 0 && ((uintptr_t)params & 7) == 0 && ((uintptr_t)tables_dev & 15) == 0,
             "resize_batch_interp: the descriptor table and params must be 8-byte aligned, the tables 16-byte aligned");
  const int rc = resize_interp_check(desc_host, images_bytes, n, new_h, new_w, letterbox, interp_host,
                                     "resize_batch_interp");
  if (rc) return rc;
  const size_t need = resize_tables_build(desc_host, n, new_h, new_w, letterbox, interp_host, nullptr);
  YB_REQUIRE(tables_bytes == need, "resize_batch_interp: tables_bytes is %zu, the tables of this call take %zu",
             tables_bytes, need);
  const ResizeTab* th = static_cast<const ResizeTab*>(tables_host);
  for (int i = 0; i < n; ++i) {
    const ResizeGeom g = resize_geom((int)desc_host[4L * i + 1], (int)desc_host[4L * i + 2], new_h, new_w, letterbox);
    YB_REQUIRE(th[i].interp == interp_host[i] && th[i].src_h == desc_host[4L * i + 1] &&
                   th[i].src_w == desc_host[4L * i + 2] && th[i].rh == g.rh && th[i].rw == g.rw,
               "resize_batch_interp: image %d: the tables were built for another image, target or interpolation", i);
  }
  const long total = (long)new_h * new_w;
  long bx = (total + 255) / 256;
  const long cap = ((long)num_sms() * 16 + n - 1) / n;  // as yb_resize_batch
  if (bx > cap) bx = cap;
  resize_batch_kernel<true><<<dim3((unsigned)bx, (unsigned)n), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      images, desc_dev, new_h, new_w, letterbox, 0, static_cast<const uint8_t*>(tables_dev), out_rgb, params);
  YB_CUDA(cudaGetLastError());
  return YB_OK;
}

extern "C" int yb_resize_boxes(float* boxes, const int32_t* counts, int n, int vmax, int box_ld, const int64_t* desc_dev,
                               int new_h, int new_w, int letterbox, void* stream) {
  YB_REQUIRE(boxes && counts && desc_dev, "resize_boxes: null pointer");
  YB_REQUIRE(((uintptr_t)desc_dev & 7) == 0, "resize_boxes: the descriptor table must be 8-byte aligned");
  YB_REQUIRE(n > 0 && vmax > 0 && box_ld >= 4, "resize_boxes: bad shape (n %d, vmax %d, box_ld %d)", n, vmax, box_ld);
  YB_REQUIRE(new_h > 0 && new_w > 0 && (letterbox == 0 || letterbox == 1), "resize_boxes: bad target or mode");
  const long total = (long)n * vmax;
  resize_boxes_kernel<<<ceil_div(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      boxes, counts, n, vmax, box_ld, desc_dev, new_h, new_w, letterbox);
  YB_CUDA(cudaGetLastError());
  return YB_OK;
}

extern "C" int yb_restore_boxes(float* boxes, const int32_t* counts, int n, int slots, int box_ld, const double* params,
                                void* stream) {
  YB_REQUIRE(boxes && counts && params, "restore_boxes: null pointer");
  YB_REQUIRE(((uintptr_t)params & 7) == 0, "restore_boxes: params must be 8-byte aligned");
  YB_REQUIRE(n > 0 && slots > 0 && box_ld >= 4, "restore_boxes: bad shape (n %d, slots %d, box_ld %d)", n, slots, box_ld);
  const long total = (long)n * slots;
  restore_boxes_kernel<<<ceil_div(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(boxes, counts, n, slots,
                                                                                            box_ld, params);
  YB_CUDA(cudaGetLastError());
  return YB_OK;
}
