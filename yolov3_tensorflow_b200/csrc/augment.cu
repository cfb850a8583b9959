// The training augmentations of parse_data(mode='train') (utils/data_utils.py:140-165 of the reference) on the device:
//   * yb_augment_batch: mix-up -> brightness -> BGR2HSV -> hue / saturation / value -> clip -> HSV2BGR -> expand ->
//     crop, fused.  Every step is per pixel or a change of placement, so each output pixel is one gather: through the
//     crop window and the expand offset to a position of the mixed image (outside it: the fill value), the mixed pixel
//     from image 1 and / or image 2, then the colour chain.  The expanded canvas is never materialised.
//   * yb_flip_batch: random_flip's horizontal / vertical flips in place on a batch of equal-size images (the resized
//     network input) and the matching box transform.
// All random draws happen on the host; the kernels see one parameter record per image.
//
// Bit-exactness notes (OpenCV 4.13, x86-64 build):
//   * BGR2HSV is the integer path with 12-bit reciprocal tables, the same in the vector and scalar code.
//   * HSV2BGR is float: 1 - s * f and 1 - s * (1 - f) are fused multiply-adds in both code paths; the vector path
//     (each row's first floor(W / 32) * 32 pixels, 32 being the AVX2 block of uint8 lanes) truncates channel * 255
//     to uint8, the scalar tail rounds it half to even.  The column rule is part of the result, so it is kept here.
#include "common.cuh"

namespace yb {

static constexpr int AUG_MAX_SIDE = 1 << 20;      // image, canvas and crop sides; keeps index products in int64
static constexpr int HSV_SIMD_PIXELS = 32;        // OpenCV's HSV2BGR vector block (AVX2: 32 uint8 lanes)
static constexpr int HSV_SHIFT = 12;

// mixed image size: image 1 alone, or the larger of both sides under a mix-up (utils/data_aug.py:18-19)
__host__ __device__ inline void mixed_size(const int64_t* desc, int src1, int src2, int& h, int& w) {
  h = (int)desc[4L * src1 + 1];
  w = (int)desc[4L * src1 + 2];
  if (src2 >= 0) {
    h = max(h, (int)desc[4L * src2 + 1]);
    w = max(w, (int)desc[4L * src2 + 2]);
  }
}

__device__ __forceinline__ int clamp255(int v) { return min(max(v, 0), 255); }

// OpenCV RGB2HSV_b (hrange 180): v = max, diff = v - min, s and h through the reciprocal tables.
__device__ __forceinline__ void bgr2hsv(int b, int g, int r, const int* sdiv, const int* hdiv, int& h, int& s, int& v) {
  v = max(max(b, g), r);
  const int diff = v - min(min(b, g), r);
  const int half = 1 << (HSV_SHIFT - 1);
  s = (diff * sdiv[v] + half) >> HSV_SHIFT;
  h = v == r ? g - b : (v == g ? b - r + 2 * diff : r - g + 4 * diff);
  h = (h * hdiv[diff] + half) >> HSV_SHIFT;
  if (h < 0) h += 180;
}

// OpenCV HSV2RGB_b (hrange 180) -> uint8 b, g, r; `simd` selects the vector path's truncation.
__device__ __forceinline__ void hsv2bgr(int hi, int si, int vi, bool simd, int& b, int& g, int& r) {
  float h = __fmul_rn((float)hi, 6.f / 180.f);
  const float s = __fmul_rn((float)si, 1.f / 255.f), v = __fmul_rn((float)vi, 1.f / 255.f);
  const float sector_f = floorf(h);
  h = __fsub_rn(h, sector_f);
  const int sector = (int)sector_f % 6;
  const float t0 = v, t1 = __fmul_rn(v, __fsub_rn(1.f, s)), t2 = __fmul_rn(v, __fmaf_rn(-s, h, 1.f)),
              t3 = __fmul_rn(v, __fmaf_rn(-s, __fsub_rn(1.f, h), 1.f));
  float tb, tg, tr;                                   // OpenCV's sector_data table
  switch (sector) {
    case 0: tb = t1; tg = t3; tr = t0; break;
    case 1: tb = t1; tg = t0; tr = t2; break;
    case 2: tb = t3; tg = t0; tr = t1; break;
    case 3: tb = t0; tg = t2; tr = t1; break;
    case 4: tb = t0; tg = t1; tr = t3; break;
    default: tb = t2; tg = t1; tr = t0; break;
  }
  const float fb = __fmul_rn(tb, 255.f), fg = __fmul_rn(tg, 255.f), fr = __fmul_rn(tr, 255.f);
  if (simd) {
    b = clamp255((int)fb); g = clamp255((int)fg); r = clamp255((int)fr);
  } else {
    b = clamp255(__float2int_rn(fb)); g = clamp255(__float2int_rn(fg)); r = clamp255(__float2int_rn(fr));
  }
}

// grid (blocks per image, n): block (bx, img) covers output pixels bx, bx + gridDim.x, ... (x 256) of image img.
__global__ void __launch_bounds__(256)
augment_kernel(const uint8_t* __restrict__ src, const int64_t* __restrict__ desc,
               const yb_augment_param* __restrict__ params, uint8_t* __restrict__ out, int64_t* __restrict__ out_desc) {
  __shared__ int s_sdiv[256], s_hdiv[256];
  __shared__ yb_augment_param s_p;
  const int img = blockIdx.y;
  {
    const int t = threadIdx.x;             // blockDim.x == 256
    s_sdiv[t] = t ? __double2int_rn((double)(255 << HSV_SHIFT) / (double)t) : 0;
    s_hdiv[t] = t ? __double2int_rn((double)(180 << HSV_SHIFT) / (6.0 * t)) : 0;
    if (t == 0) s_p = params[img];
  }
  __syncthreads();
  const yb_augment_param p = s_p;
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    int64_t* d = out_desc + 4L * img;
    d[0] = p.out_offset; d[1] = p.out_h; d[2] = p.out_w; d[3] = 3L * p.out_w;
  }
  int mh, mw;
  mixed_size(desc, p.src1, p.src2, mh, mw);
  const int64_t* d1 = desc + 4L * p.src1;
  const uint8_t* im1 = src + d1[0];
  const int h1 = (int)d1[1], w1 = (int)d1[2];
  const long pitch1 = (long)d1[3];
  const uint8_t* im2 = im1;
  int h2 = 0, w2 = 0;
  long pitch2 = 0;
  if (p.src2 >= 0) {
    const int64_t* d2 = desc + 4L * p.src2;
    im2 = src + d2[0]; h2 = (int)d2[1]; w2 = (int)d2[2]; pitch2 = (long)d2[3];
  }
  const int simd_cols = mw - mw % HSV_SIMD_PIXELS;
  uint8_t* o = out + p.out_offset;
  const long total = (long)p.out_h * p.out_w;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int oy = (int)(i / p.out_w), ox = (int)(i - (long)oy * p.out_w);
    const int my = oy + p.crop_y - p.off_y, mx = ox + p.crop_x - p.off_x;
    int c[3] = {p.fill, p.fill, p.fill};
    if (my >= 0 && my < mh && mx >= 0 && mx < mw) {
      if (p.src2 < 0) {
        const uint8_t* q = im1 + (long)my * pitch1 + 3L * mx;
        c[0] = q[0]; c[1] = q[1]; c[2] = q[2];
      } else {
        // mix_up: float32 img1 * w1 stored, img2 * w2 added where it lies, truncated (utils/data_aug.py:21-29)
        const bool in1 = my < h1 && mx < w1, in2 = my < h2 && mx < w2;
        const uint8_t* q1 = im1 + (long)my * pitch1 + 3L * mx;
        const uint8_t* q2 = im2 + (long)my * pitch2 + 3L * mx;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          const float a = in1 ? __fmul_rn((float)q1[k], p.w1) : 0.f;
          const float b = in2 ? __fmul_rn((float)q2[k], p.w2) : 0.f;
          c[k] = (int)__fadd_rn(a, b);
        }
      }
      if (p.color) {
        // random_brightness: float32 + int delta, clip, truncate; then the HSV round trip with the drawn ops
        int h, s, v;
        bgr2hsv(clamp255(c[0] + p.brightness), clamp255(c[1] + p.brightness), clamp255(c[2] + p.brightness), s_sdiv,
                s_hdiv, h, s, v);
        h = (h + p.hue) % 180;                              // np.remainder: the sign of the divisor
        if (h < 0) h += 180;
        s = (int)fminf(fmaxf(__fmul_rn((float)s, p.saturation), 0.f), 255.f);
        v = (int)fminf(fmaxf(__fmul_rn((float)v, p.value), 0.f), 255.f);
        hsv2bgr(h, s, v, mx < simd_cols, c[0], c[1], c[2]);
      }
    }
    uint8_t* q = o + 3 * i;
    q[0] = (uint8_t)c[0]; q[1] = (uint8_t)c[1]; q[2] = (uint8_t)c[2];
  }
}

// random_flip in place: pixel i and its mirror swap once (the lower index does it).  Block column 0 also flips the
// image's boxes: x' = W - x with min and max swapped (y likewise), float32.
template <typename T>
__global__ void __launch_bounds__(256)
flip_kernel(T* __restrict__ x, int h, int w, const int32_t* __restrict__ flags, float* __restrict__ boxes,
            const int32_t* __restrict__ counts, int vmax, int ld) {
  const int img = blockIdx.y;
  const int f = flags[img];
  if (!(f & 3)) return;
  const bool fx = f & 1, fy = f & 2;
  if (boxes && blockIdx.x == 0) {
    const int cnt = min(counts[img], vmax);
    const float W = (float)w, H = (float)h;
    for (int j = threadIdx.x; j < cnt; j += blockDim.x) {
      float* b = boxes + ((long)img * vmax + j) * ld;
      if (fx) { const float x0 = b[0]; b[0] = __fsub_rn(W, b[2]); b[2] = __fsub_rn(W, x0); }
      if (fy) { const float y0 = b[1]; b[1] = __fsub_rn(H, b[3]); b[3] = __fsub_rn(H, y0); }
    }
  }
  T* im = x + (long)img * h * w * 3;
  const long total = (long)h * w;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int y = (int)(i / w), xx = (int)(i - (long)y * w);
    const long j = (long)(fy ? h - 1 - y : y) * w + (fx ? w - 1 - xx : xx);
    if (j <= i) continue;
    T* a = im + 3 * i;
    T* b = im + 3 * j;
#pragma unroll
    for (int k = 0; k < 3; ++k) { const T t = a[k]; a[k] = b[k]; b[k] = t; }
  }
}

}  // namespace yb

using namespace yb;

extern "C" int yb_augment_batch(const uint8_t* images, long images_bytes, const int64_t* desc_host,
                                const int64_t* desc_dev, int n_in, const yb_augment_param* params_host,
                                const yb_augment_param* params_dev, int n, uint8_t* out, long out_bytes,
                                int64_t* out_desc_dev, void* stream) {
  YB_REQUIRE(images && desc_host && desc_dev && params_host && params_dev && out && out_desc_dev,
             "augment_batch: null pointer");
  YB_REQUIRE(((uintptr_t)desc_dev & 7) == 0 && ((uintptr_t)params_dev & 7) == 0 && ((uintptr_t)out_desc_dev & 7) == 0,
             "augment_batch: the descriptor tables and the parameter table must be 8-byte aligned");
  YB_REQUIRE(n_in > 0 && n > 0 && n <= 65535, "augment_batch: need 1..65535 outputs from >= 1 inputs (got %d, %d)", n,
             n_in);
  for (int i = 0; i < n_in; ++i) {
    const int64_t off = desc_host[4L * i], h = desc_host[4L * i + 1], w = desc_host[4L * i + 2],
                  pitch = desc_host[4L * i + 3];
    YB_REQUIRE(h > 0 && w > 0 && h <= AUG_MAX_SIDE && w <= AUG_MAX_SIDE, "augment_batch: image %d has size %lldx%lld",
               i, (long long)w, (long long)h);
    YB_REQUIRE(off >= 0 && pitch >= 3 * w && off + (h - 1) * pitch + 3 * w <= images_bytes,
               "augment_batch: image %d (offset %lld, pitch %lld) lies outside the %ld-byte buffer", i, (long long)off,
               (long long)pitch, images_bytes);
  }
  long work = 0;
  for (int i = 0; i < n; ++i) {
    const yb_augment_param& p = params_host[i];
    YB_REQUIRE(p.src1 >= 0 && p.src1 < n_in && p.src2 >= -1 && p.src2 < n_in,
               "augment_batch: output %d reads images %d / %d of %d", i, p.src1, p.src2, n_in);
    int mh, mw;
    mixed_size(desc_host, p.src1, p.src2, mh, mw);
    YB_REQUIRE(p.canvas_h >= mh && p.canvas_w >= mw && p.canvas_h <= AUG_MAX_SIDE && p.canvas_w <= AUG_MAX_SIDE,
               "augment_batch: output %d: canvas %dx%d cannot hold the %dx%d image", i, p.canvas_w, p.canvas_h, mw, mh);
    YB_REQUIRE(p.off_y >= 0 && p.off_x >= 0 && p.off_y <= p.canvas_h - mh && p.off_x <= p.canvas_w - mw,
               "augment_batch: output %d: expand offset (%d, %d) puts the image outside the canvas", i, p.off_x,
               p.off_y);
    YB_REQUIRE(p.out_h >= 0 && p.out_w >= 0 && p.crop_y >= 0 && p.crop_x >= 0 && p.crop_y <= p.canvas_h - p.out_h &&
                   p.crop_x <= p.canvas_w - p.out_w,
               "augment_batch: output %d: crop (%d, %d, %d, %d) lies outside the %dx%d canvas", i, p.crop_x, p.crop_y,
               p.out_w, p.out_h, p.canvas_w, p.canvas_h);
    YB_REQUIRE(p.out_offset >= 0 && p.out_offset + 3L * p.out_h * p.out_w <= out_bytes,
               "augment_batch: output %d (offset %lld) lies outside the %ld-byte output", i, (long long)p.out_offset,
               out_bytes);
    YB_REQUIRE(p.color == 0 || p.color == 1, "augment_batch: output %d: color must be 0 or 1", i);
    YB_REQUIRE(p.fill >= 0 && p.fill <= 255, "augment_batch: output %d: fill %d is not a uint8", i, p.fill);
    YB_REQUIRE(p.brightness >= -255 && p.brightness <= 255 && p.hue > -(1 << 24) && p.hue < (1 << 24),
               "augment_batch: output %d: brightness %d or hue %d out of range", i, p.brightness, p.hue);
    YB_REQUIRE(isfinite(p.w1) && isfinite(p.w2) && isfinite(p.saturation) && isfinite(p.value),
               "augment_batch: output %d: non-finite weight or multiplier", i);
    const long px = (long)p.out_h * p.out_w;
    if (px > work) work = px;
  }
  long bx = (work + 255) / 256;
  const long cap = ((long)num_sms() * 16 + n - 1) / n;  // about 16 CTAs per SM over the batch, then grid-stride
  if (bx > cap) bx = cap;
  augment_kernel<<<dim3((unsigned)bx, (unsigned)n), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      images, desc_dev, params_dev, out, out_desc_dev);
  YB_CUDA(cudaGetLastError());
  return YB_OK;
}

extern "C" int yb_flip_batch(void* x, int n, int h, int w, int elem_bytes, const int32_t* flags_dev, float* boxes,
                             const int32_t* counts, int vmax, int box_ld, void* stream) {
  YB_REQUIRE(x && flags_dev, "flip_batch: null pointer");
  YB_REQUIRE(n > 0 && n <= 65535 && h > 0 && w > 0 && h <= AUG_MAX_SIDE && w <= AUG_MAX_SIDE,
             "flip_batch: bad shape (n %d, %dx%d)", n, w, h);
  YB_REQUIRE(elem_bytes == 1 || elem_bytes == 4, "flip_batch: elements must be uint8 or float32 (got %d bytes)",
             elem_bytes);
  YB_REQUIRE(((uintptr_t)x & (elem_bytes - 1)) == 0 && ((uintptr_t)flags_dev & 3) == 0,
             "flip_batch: misaligned images or flags");
  if (boxes) {
    YB_REQUIRE(counts && vmax > 0 && box_ld >= 4, "flip_batch: boxes need counts, vmax > 0 and box_ld >= 4");
    YB_REQUIRE(((uintptr_t)boxes & 3) == 0 && ((uintptr_t)counts & 3) == 0, "flip_batch: misaligned boxes or counts");
  }
  long bx = ((long)h * w + 255) / 256;
  const long cap = ((long)num_sms() * 16 + n - 1) / n;
  if (bx > cap) bx = cap;
  const dim3 grid((unsigned)bx, (unsigned)n);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (elem_bytes == 1)
    flip_kernel<uint8_t><<<grid, 256, 0, st>>>(static_cast<uint8_t*>(x), h, w, flags_dev, boxes, counts, vmax, box_ld);
  else
    flip_kernel<float><<<grid, 256, 0, st>>>(static_cast<float*>(x), h, w, flags_dev, boxes, counts, vmax, box_ld);
  YB_CUDA(cudaGetLastError());
  return YB_OK;
}
