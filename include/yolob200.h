/* yolob200.h — C ABI of libyolob200.so: the H100-native (sm_90a) replacement for the
 * TensorFlow ops that wizyoung/YOLOv3_TensorFlow's hot path builds its graph from.
 *
 * The reference has no FFI layer of its own (it is pure Python over TensorFlow), so
 * each entry point below names the reference *call site* (file:line, relative to the
 * reference repo) whose TF ops it replaces.  The Python package
 * `yolov3_tensorflow_b200` binds these with ctypes and re-exposes the reference's
 * Python API (model.yolov3, utils.nms_utils.gpu_nms, utils.misc_utils.load_weights).
 *
 * Conventions
 *   - every function returns YB_OK (0) or a negative yb_status; text via
 *     yb_last_error_string() (thread-local).
 *   - the CALLER owns every buffer (inputs, outputs, workspaces, arenas); nothing is
 *     allocated or freed on the device behind the caller's back.
 *   - all work is enqueued on the cudaStream_t passed as `stream` (void*); no entry
 *     point synchronises the device unless its comment says so.
 *   - device pointers unless marked "host".  Activations are NHWC.
 */
#ifndef YOLOB200_H_
#define YOLOB200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum yb_status {
  YB_OK = 0,
  YB_ERR_INVALID_ARGUMENT = -1,
  YB_ERR_CUDA = -2,
  YB_ERR_UNSUPPORTED = -3,
  YB_ERR_WORKSPACE = -4
} yb_status;

/* YB_E4M3: fp8 e4m3 (OCP "fn": finite, max 448) with float32 scales, for the calibrated inference plan only */
typedef enum yb_dtype { YB_F16 = 0, YB_BF16 = 1, YB_F32 = 2, YB_E4M3 = 3 } yb_dtype;

/* layout of a conv weight tensor handed to the packer */
typedef enum yb_wlayout {
  YB_W_HWIO = 0, /* TensorFlow variable layout [kh,kw,Cin,Cout] (utils/misc_utils.py:120)   */
  YB_W_OIHW = 1, /* darknet .weights stream layout (Cout,Cin,kh,kw) (utils/misc_utils.py:117) */
  YB_W_OHWI = 2  /* engine layout [Cout,kh,kw,Cin] (K-major for the implicit GEMM)           */
} yb_wlayout;

int yb_version(void);
const char* yb_last_error_string(void);
/* Runtime switches for A/B experiments and tests (DESIGN.md 5b: "YB_HALO", "YB_STEM_FUSE", ...).  The table is
 * seeded once from the equally named environment variables when the library is first used; afterwards only
 * yb_set_option() changes it (value NULL or "" = default).  No entry point calls getenv() on its own. */
int yb_set_option(const char* key, const char* value);
const char* yb_get_option(const char* key);
/* device 0..: SM count and compute capability of the current device. */
int yb_device_info(int* sm_count, int* cc_major, int* cc_minor);

/* ---------------------------------------------------------------------------------
 * Convolution  (replaces slim.conv2d + slim.batch_norm + leaky_relu + tf.add +
 * tf.pad + resize_nearest_neighbor + tf.concat: utils/layer_utils.py:9-22,30,82-87,
 * model.py:43-49,55-57,62,72)
 * --------------------------------------------------------------------------------- */
typedef struct yb_conv_desc {
  int n, h, w;      /* input batch / height / width                                         */
  int cin, cout;    /* real channel counts (cout = 255 for the detection heads)             */
  int ksize;        /* 1 or 3                                                               */
  int stride;       /* 1 (SAME) or 2 (pad 1 each side then VALID — darknet rule)            */
  int in_ld;        /* elements between consecutive input pixels  (>= cin; concat slices)   */
  int out_ld;       /* elements between consecutive output pixels (>= cout)                 */
  int res_ld;       /* same for the residual input (ignored when res == NULL)               */
  int dtype;        /* yb_dtype of x / w / res (and of out unless out_fp32)                 */
  int out_fp32;     /* 1: write float32 (detection heads), 0: write `dtype`                 */
  int leaky;        /* 1: leaky_relu(0.1) after scale/shift                                 */
  int upsample2x;   /* 1: nearest-neighbour 2x: every output pixel is stored to its 4 places
                          in an [n, 2*ho, 2*wo, out_ld] buffer (model.py:61,71)             */
} yb_conv_desc;

/* Epilogue note (round 2): 16-bit outputs leave each CTA through swizzled shared memory and cp.async.bulk.tensor
 * (TMA) stores, the residual arrives by TMA into the same staging tile; scale = shift = NULL means identity.
 *
 * out[p, co] = act( scale[co] * sum_{r,s,ci} x[p*stride + (r,s) - pad, ci] * w[co,r,s,ci] + shift[co] ) (+ res[p, co])
 *   x        [n,h,w,in_ld]   dtype
 *   w_packed [cout_pad, ksize, ksize, cin] dtype, cout_pad = yb_conv_cout_pad(cout) (zero rows beyond cout)
 *   scale, shift  float32 [cout_pad]   (BN folded: gamma/sqrt(var+eps), beta-mean*scale; heads: 1, bias)
 *   res      nullable, [n,ho,wo,res_ld] dtype — added AFTER the activation (utils/layer_utils.py:30)
 *   out      [n,ho,wo,out_ld] (or the 2x-upsampled buffer)
 *   stat_sum/stat_sqsum nullable float32 [cout_pad]: when given, the per-channel sum and sum of squares of
 *            the raw convolution result (before scale/shift) are atomically accumulated (BN batch statistics).
 * Requires cin % 32 == 0 (the 3-channel stem has its own entry point).  wgmma implicit GEMM. */
int yb_conv2d_fwd(const yb_conv_desc* d, const void* x, const void* w_packed, const float* scale,
                  const float* shift, const void* res, void* out, float* stat_sum, float* stat_sqsum,
                  void* stream);
int yb_conv_cout_pad(int cout);
/* e4m3 form of yb_conv2d_fwd (d->dtype = YB_E4M3; the fp8 inference plan's convs): x, w_packed and res hold e4m3 codes,
 * value = code x scale.  scale[co] must already carry (BN scale) x (input scale) x (weight scale of channel co);
 * out = e4m3 codes of value / out_scale (RN, saturating to +-448), or float32 values when d->out_fp32.  The residual
 * is added as code x res_scale after the activation.  cin % 64 == 0 and in_ld, out_ld, res_ld multiples of 16; no
 * statistics.  Runs the ping-pong and cooperative schedules (YB_CONV_PP, YB_CONV_CTAS apply); YB_CONV_EG=1,
 * YB_CONV_MODE=2cta and YB_CONV_EPI=reg return YB_ERR_INVALID_ARGUMENT. */
int yb_conv2d_fwd_e4m3(const yb_conv_desc* d, const void* x, const void* w_packed, const float* scale,
                       const float* shift, const void* res, float res_scale, void* out, float out_scale, void* stream);
/* Host-only: the implicit-GEMM kernel and persistent grid yb_conv2d_fwd would launch for `d` with the current options
 * (yb_set_option: YB_CONV_EG, YB_CONV_MODE, YB_CONV_EPI, YB_CONV_PP, YB_CONV_CTAS) on a device with sm_count SMs.
 * kh = kw = 0: the forward ksize x ksize window; kh, kw in {1, 2}: one parity class of yb_conv2d_dgrad_s2 (d = its
 * stride-1 descriptor over dz).  with_stats: BN statistics requested.  The clusters of the grid take the work units
 * round-robin, and under ping-pong the two consumer warpgroups of a CTA take every other one of its cluster's units. */
typedef struct yb_conv_schedule_info {
  int pingpong;      /* 1: ping-pong (each consumer warpgroup owns whole tiles), 0: cooperative */
  int consumers;     /* consumer warpgroups per CTA                                             */
  int cluster;       /* CTAs per cluster                                                        */
  int block_m, block_n, block_k;
  int stages;        /* operand-ring depth                                                      */
  int num_kb;        /* k-blocks per tile                                                       */
  int num_m_tiles, num_n_tiles;
  int grid;          /* CTAs launched                                                           */
  int res_smem;      /* 1: a launch with a residual prefetches it into shared memory (YB_CONV_RES) */
  int res_stages;    /* operand-ring depth of a launch with a residual                          */
  int cluster_m;     /* CTAs of a cluster along M (each a different m-tile)                     */
  int cluster_n;     /* CTAs of a cluster along N (1 | 2; 1 under the cooperative schedule)     */
  int units;         /* work units: ceil(num_m_tiles / cluster_m) x num_n_tiles / cluster_n     */
  int epi_tma;       /* 1: the epilogue packs the accumulator fragments to 16 bits and stores them by TMA */
                     /*    (YB_CONV_EPI=tma, or unset in a 16-bit inference plan); 0: staged or register. */
                     /*    A launch with a residual takes it only if res_smem                             */
} yb_conv_schedule_info;
int yb_conv_schedule(const yb_conv_desc* d, int kh, int kw, int with_stats, int sm_count, yb_conv_schedule_info* info);

/* First layer (darknet53_body/Conv, 3->32, 3x3 s1; utils/layer_utils.py:35): float32 NHWC image in,
 * `dtype` NHWC out.  w is OHWI float32 [32,3,3,3]. */
int yb_stem_conv_fwd(const float* x, const float* w_ohwi, const float* scale, const float* shift, int n, int h,
                     int w, int cout, int dtype, int leaky, void* out, void* stream);

/* Thin-layer fast paths (HBM-bound layers at the top of Darknet-53; see csrc/conv_thin.cu): same contract as
 * yb_conv2d_fwd / yb_stem_conv_fwd, restricted to 3x3, cin = 32, cout in {32,64} (no statistics, 16-bit output),
 * resp. the 3->32 stem.  Halo tile + resident weights in shared memory, warp-level tensor path. */
int yb_conv3x3_thin_fwd(const yb_conv_desc* d, const void* x, const void* w_packed, const float* scale,
                        const float* shift, const void* res, void* out, void* stream);
int yb_stem_conv_fwd_tc(const float* x, const float* w_ohwi, const float* scale, const float* shift, int n, int h,
                        int w, int dtype, int leaky, void* out, void* stream);
/* ... and, for the training forward, also ACCUMULATING the per-channel sum / sum of squares of the stored outputs
 * (fp32 [32] each, zeroed by the caller; both NULL = yb_stem_conv_fwd_tc): the batch statistics of
 * slim.batch_norm(is_training=True) (reference model.py:35-41) without a second pass over the tensor. */
int yb_stem_conv_fwd_tc_stats(const float* x, const float* w_ohwi, const float* scale, const float* shift, int n, int h,
                              int w, int dtype, int leaky, void* out, float* stat_sum, float* stat_sqsum, void* stream);

/* 3x3 convs with cin in {32, 64} and cout in {64, 128}, except 64 -> 128 at stride 2 (darknet53_body Conv_1/3/6/8,
 * utils/layer_utils.py:36-44) from a shared-memory HALO tile: one tiled TMA load per 16x8-pixel output tile (four parity
 * planes for stride 2), the nine taps are nine wgmma descriptors into that tile, weights resident in shared memory
 * (csrc/conv_halo.cu).  Same contract as yb_conv2d_fwd without statistics; fp16 / bf16, 16-bit output;
 * (w / stride) % 8 == 0.  yb_conv3x3_halo_supported: 1 if d fits. */
int yb_conv3x3_halo_supported(const yb_conv_desc* d);
int yb_conv3x3_halo_fwd(const yb_conv_desc* d, const void* x, const void* w_packed, const float* scale,
                        const float* shift, const void* res, void* out, void* stream);
/* darknet53_body/Conv (3->32, 3x3/1) fused into darknet53_body/Conv_1 (32->64, 3x3/2) (utils/layer_utils.py:35-36):
 * the stem is computed on the fly as the producer of Conv_1's shared-memory halo planes, its 64 B/pixel output is never
 * written.  image float32 [n, h, w, 3]; d describes Conv_1 (d->h, d->w = image size, cin 32, cout 64, stride 2);
 * stem_w_ohwi float32 [32][27], stem_scale / stem_shift float32 [32] (folded BN); out [n, h/2, w/2, out_ld] 16-bit. */
int yb_stem_conv1_fused_fwd(const yb_conv_desc* d, const float* image, const float* stem_w_ohwi, const float* stem_scale,
                            const float* stem_shift, const void* w_packed, const float* scale, const float* shift, void* out,
                            void* stream);

/* ---------------------------------------------------------------------------------
 * Pre-processing either side of the hot path, on the device (SURVEY.md 8f N3)
 * --------------------------------------------------------------------------------- */
/* process_box (utils/data_utils.py:51-115) for a batch: ground-truth lists -> y_true_13/26/52.
 *   boxes  float32 [n, vmax, 5] (x_min, y_min, x_max, y_max, mixup weight), labels int32 [n, vmax], counts int32 [n]
 *   (boxes beyond counts[i] are ignored); anchors9x2 host float[18]; y_true_s float32 [n, h/s, w/s, 3, 6 + class_num],
 *   fully overwritten (zeros, mix weight 1, then the boxes in list order: the last box of a slot wins, class bits
 *   accumulate — exactly the reference's loop).  Bit-exact vs the reference.  vmax <= 256. */
int yb_process_box(const float* boxes, const int32_t* labels, const int32_t* counts, int n, int vmax, int img_w,
                   int img_h, int class_num, const float* anchors9x2, float* y_true_1, float* y_true_2,
                   float* y_true_3, void* stream);
/* letterbox_resize(img, new_w, new_h, interp=0) (utils/data_aug.py:274-293) + BGR->RGB + float32 / 255
 * (test_single_image.py:39-46): uint8 BGR [src_h, src_w, 3] (row pitch in bytes) -> float32 RGB [new_h, new_w, 3].
 * yb_letterbox_params returns the host-side scalars of the same call (resize_ratio, resized size, dh, dw). */
int yb_letterbox_params(int src_h, int src_w, int new_h, int new_w, double* resize_ratio, int* resize_h, int* resize_w,
                        int* dh, int* dw);
int yb_letterbox_normalize(const uint8_t* bgr, int src_h, int src_w, long src_pitch_bytes, int new_h, int new_w,
                           float* out_rgb, void* stream);
/* The evaluation input path for a batch of images of different sizes, in one launch: letterbox_resize or a plain
 * stretch (cv2.resize to the target), nearest (interp 0) or OpenCV's bilinear (interp 1), then BGR->RGB + float32 / 255
 * (parse_data(mode='val') at utils/data_utils.py:166-176, eval.py, test_single_image.py:39-46).
 *   images     device, n uint8 BGR images packed in images_bytes bytes
 *   desc_host  host int64 [n, 4]: (byte offset, h, w, row pitch in bytes) per image, validated here;
 *   desc_dev   the same table on the device (8-byte aligned), read by the kernel: the two must hold the same values
 *   out_rgb    float32 [n, new_h, new_w, 3]; letterbox borders are 128 / 255
 *   params     optional float64 [n, 4]: letterbox (resize_ratio, dw, dh, 1), stretch (w / new_w, h / new_h, 0, 0)
 * Bit-exact vs cv2.resize of OpenCV 4.13 (INTER_LINEAR is not bit-stable across OpenCV builds).  n <= 65535, image
 * sides in 1..2^20, and a letterbox whose int() truncation leaves an empty resize is rejected. */
int yb_resize_batch(const uint8_t* images, long images_bytes, const int64_t* desc_host, const int64_t* desc_dev, int n,
                    int new_h, int new_w, int letterbox, int interp, float* out_rgb, double* params, void* stream);
/* The training resize (parse_data(mode='train'), utils/data_utils.py:160-161: resize_with_bbox with the drawn
 * interp): yb_resize_batch with one OpenCV interpolation per image, interp_host int32 [n] in 0..4 -- 0 nearest,
 * 1 linear (both equal to yb_resize_batch's output), 2 INTER_CUBIC, 3 INTER_AREA, 4 INTER_LANCZOS4.  Each image's
 * per-axis tap tables are built on the host as OpenCV builds them (Lanczos4 from the C library's sin / cos) into one
 * 16-byte aligned buffer: yb_resize_tables_bytes gives its size, yb_resize_tables fills it (host only, no device
 * work), the caller copies it to the device and passes both copies to yb_resize_batch_interp (the host copy is checked
 * against the call).  A 608 x 608 cubic / Lanczos4 / upscaling area table is 24 kB; a shrinking area table holds
 * 8 bytes per destination index and up to 16 per source index.
 * Bit-exact vs cv2.resize of OpenCV 4.13 for INTER_AREA and INTER_LANCZOS4, and for INTER_CUBIC vs OpenCV's own code
 * (cv2.ipp.setUseIPP(False)); default cv2 builds send uint8 INTER_CUBIC through Intel IPP, which differs by at most 1.
 * Same size in and out is a copy.  Everything is validated before any device work. */
int yb_resize_tables_bytes(const int64_t* desc_host, int n, int new_h, int new_w, int letterbox,
                           const int32_t* interp_host, size_t* bytes);
int yb_resize_tables(const int64_t* desc_host, int n, int new_h, int new_w, int letterbox, const int32_t* interp_host,
                     void* tables_host, size_t bytes);
int yb_resize_batch_interp(const uint8_t* images, long images_bytes, const int64_t* desc_host, const int64_t* desc_dev,
                           int n, int new_h, int new_w, int letterbox, const int32_t* interp_host,
                           const void* tables_host, const void* tables_dev, size_t tables_bytes, float* out_rgb,
                           double* params, void* stream);
/* resize_with_bbox's box transform (utils/data_aug.py:301-318), in place, float32 in the reference's order:
 * boxes float32 [n, vmax, box_ld] (columns 0-3 x_min, y_min, x_max, y_max; the rest untouched), counts int32 [n],
 * desc_dev the yb_resize_batch descriptor table of the same images. */
int yb_resize_boxes(float* boxes, const int32_t* counts, int n, int vmax, int box_ld, const int64_t* desc_dev, int new_h,
                    int new_w, int letterbox, void* stream);
/* Detections back to source-image coordinates (test_single_image.py:64-70), in place: boxes float32 [n, slots, box_ld]
 * (yb_net_detect's per-image output slots), the first counts[i] of image i mapped with params row i of yb_resize_batch. */
int yb_restore_boxes(float* boxes, const int32_t* counts, int n, int slots, int box_ld, const double* params,
                     void* stream);

/* ---------------------------------------------------------------------------------
 * Training augmentation  (replaces parse_data(mode='train')'s image work around the resize, utils/data_utils.py:
 * 140-165: mix_up, random_color_distort, random_expand, the crop of random_crop_with_constraints and random_flip)
 * --------------------------------------------------------------------------------- */
/* One output image of yb_augment_batch.  All random draws are made on the host; this is what they decided. */
typedef struct yb_augment_param {
  int64_t out_offset;          /* byte offset of the output image in `out`                              */
  int32_t out_h, out_w;        /* crop size = output size                                               */
  int32_t crop_y, crop_x;      /* crop origin on the canvas                                             */
  int32_t canvas_h, canvas_w;  /* expanded canvas; the mixed image's size when not expanded             */
  int32_t off_y, off_x;        /* origin of the mixed image on the canvas                               */
  int32_t src1, src2;          /* input images; src2 = -1: no mix-up                                    */
  float w1, w2;                /* mix-up weights float32(r), float32(1 - r)                             */
  int32_t color;               /* 1: brightness + BGR2HSV + hue / saturation / value + HSV2BGR          */
  int32_t brightness;          /* delta added before BGR2HSV (0: not drawn)                             */
  int32_t hue;                 /* delta added to H, mod 180 (0: not drawn)                              */
  float saturation, value;     /* multipliers of S and V (1: not drawn)                                 */
  int32_t fill;                /* canvas value outside the mixed image, 0..255                          */
} yb_augment_param;
/* mix-up -> brightness -> BGR2HSV -> hue / saturation / value -> clip -> HSV2BGR -> expand -> crop in one launch:
 * images / desc_host / desc_dev as yb_resize_batch (n_in inputs), params_host and params_dev the same n records
 * (host copy for validation, device copy for the kernel), out the output pixels, out_desc_dev the output's int64
 * [n, 4] descriptor table (offset, h, w, 3 w), written by the kernel.  Pixels equal OpenCV 4.13's cvtColor (x86-64
 * build: vector blocks of 32 pixels truncate in HSV2BGR, the scalar row tail rounds) and numpy's float32 arithmetic.
 * Descriptors, image indices, expand offsets, crop windows and output ranges are checked before any device work. */
int yb_augment_batch(const uint8_t* images, long images_bytes, const int64_t* desc_host, const int64_t* desc_dev,
                     int n_in, const yb_augment_param* params_host, const yb_augment_param* params_dev, int n,
                     uint8_t* out, long out_bytes, int64_t* out_desc_dev, void* stream);
/* random_flip in place on n equal-size images x [n, h, w, 3] of uint8 (elem_bytes 1) or float32 (4): flags_dev int32
 * [n], bit 0 horizontal (cv2.flip(img, 1)), bit 1 vertical (cv2.flip(img, 0)).  With boxes (float32 [n, vmax,
 * box_ld], the first counts[i] of image i): x' = w - x, y' = h - y with min and max swapped, float32.  One launch. */
int yb_flip_batch(void* x, int n, int h, int w, int elem_bytes, const int32_t* flags_dev, float* boxes,
                  const int32_t* counts, int vmax, int box_ld, void* stream);

/* Weight repack (utils/misc_utils.py:114-123 does (Cout,Cin,kh,kw) -> HWIO on the host):
 * src float32 in `layout` -> dst `dtype` (or float32) OHWI [cout_pad,k,k,cin], rows >= cout zeroed. */
int yb_pack_conv_weights(const float* src, int layout, int cout, int cin, int ksize, int cout_pad, int dtype,
                         void* dst, void* stream);
/* Same repack to e4m3 with per-output-channel scales: w_scale[co] (float32 [cout_pad]) = max_k |w[co, k]| / 448 and
 * dst[co, k] = RN-satfinite e4m3(w[co, k] / w_scale[co]); rows whose max is 0 (and the padding rows >= cout) get
 * scale 1 and zero codes. */
int yb_pack_conv_weights_e4m3(const float* src, int layout, int cout, int cin, int ksize, int cout_pad, void* dst,
                              float* w_scale, void* stream);
/* out (device float[1], overwritten) = max |x| over the strided [rows, cols] matrix x (row pitch ld elements, dtype
 * f16 / bf16 / f32): the calibration statistic of the fp8 plan.  Exact, hence bit-reproducible. */
int yb_amax(const void* x, long ld, long rows, int cols, int dtype, float* out, void* stream);
/* BN inference fold (model.py:35-41, eps=1e-5): scale = gamma/sqrt(var+eps), shift = beta - mean*scale. */
int yb_bn_fold(const float* gamma, const float* beta, const float* mean, const float* var, int c, float eps,
               float* scale, float* shift, void* stream);

/* ---------------------------------------------------------------------------------
 * Training-mode pieces around the conv (replace slim.batch_norm(is_training=True) and TF autodiff of
 * slim.conv2d / batch_norm / leaky_relu: model.py:35-49, train.py:108-112)
 * --------------------------------------------------------------------------------- */
/* dw[cout, k*k*cin] (fp32, OHWI, ACCUMULATED) += sum over output pixels of dz[p,co] * im2col(x)[p,(r,s,ci)].
 * d describes the FORWARD conv (n,h,w,cin,cout,ksize,stride,in_ld,dtype); x is its input activation,
 * dz [n*ho*wo, dz_ld] the gradient w.r.t. its raw output; dz_dilated=1: dz is stored zero-inserted in an
 * [n, 2ho, 2wo, dz_ld] buffer (what the stride-2 dgrad consumes).  wgmma, MN-major operands, split over pixels. */
int yb_conv2d_wgrad(const yb_conv_desc* d, const void* x, const void* dz, int dz_ld, int dz_dilated, float* dw,
                    void* stream);
/* wgrad of the 3-channel stem: x float32 [n,h,w,3], dz [n*h*w, 32] 16-bit -> dw [32,3,3,3] accumulated. */
int yb_stem_conv_wgrad(const float* x, const void* dz, int dtype, int n, int h, int w, float* dw, void* stream);
/* Same contract on the warp-level tensor path (image split into 16-bit head + remainder: float32-exact to ~1e-5);
 * yb_stem_conv_wgrad dispatches to it by default. */
int yb_stem_conv_wgrad_tc(const float* x, const void* dz, int dtype, int n, int h, int w, float* dw, void* stream);
/* dgrad weights: dst[ci][r][s][co] = w_ohwi[co][k-1-r][k-1-s][ci] (k_cout >= cout, cin_pad >= cin zero-padded):
 * the data gradient of a stride-1 conv is yb_conv2d_fwd(dz, dst) (stride-2: on the zero-inserted dz). */
int yb_pack_dgrad_weights(const float* w_ohwi, int cout, int cin, int ksize, int k_cout, int cin_pad, int dtype,
                          void* dst, void* stream);
/* Data gradient of a 3x3 STRIDE-2 conv (pad 1 + VALID, utils/layer_utils.py:17-27) without zero insertion: the input
 * pixels are split by parity (a, b) = (row & 1, col & 1); class (a, b) is a (1+a) x (1+b)-tap conv over the plain
 * dz [n, h/2, w/2, dz_ld] whose result is stored at (2i + a, 2j + b) of dx [n, h, w, dx_ld] (+ res at the same pixel,
 * res nullable, may alias dx).  yb_pack_dgrad_weights_s2 lays the four weight matrices [cin_pad][(1+a)(1+b)*k_cout]
 * out back to back (9 * cin_pad * k_cout elements).  `fwd` is the FORWARD conv's descriptor (n, h, w, cin, cout, dtype). */
int yb_pack_dgrad_weights_s2(const float* w_ohwi, int cout, int cin, int k_cout, int cin_pad, int dtype, void* dst,
                             void* stream);
int yb_conv2d_dgrad_s2(const yb_conv_desc* fwd, const void* dz, int dz_ld, int k_cout, const void* w_dgrad_s2,
                       const void* res, int res_ld, void* dx, int dx_ld, void* stream);
/* Host-only: the kernel and grid yb_conv2d_wgrad would launch for `d` with the current options (yb_set_option:
 * YB_WGRAD_TP, YB_WGRAD_EPI, YB_WGRAD_SPLITS) on a device with sm_count SMs.  The output pixels form num_kb 64-pixel
 * blocks; split-K cuts them into `splits` ranges of kb_per_split blocks (the last range may be shorter, none is empty),
 * by default the count that minimises waves x (blocks per CTA + YB_WGRAD_EPI).  Grid = (splits, tap groups x input-
 * channel chunks of bnw, 128-row output-channel tiles); tiles = grid_y x grid_z. */
typedef struct yb_wgrad_schedule_info {
  int bnw;           /* input channels per tap and tile                 */
  int tp;            /* filter taps per CTA (1, or 3: one kernel row)   */
  int stages;        /* operand-ring depth of that kernel               */
  int num_kb;        /* 64-pixel blocks                                 */
  int kb_per_split;  /* blocks per CTA                                  */
  int splits;
  int tiles;
  int grid_x, grid_y, grid_z;
} yb_wgrad_schedule_info;
int yb_wgrad_schedule(const yb_conv_desc* d, int sm_count, yb_wgrad_schedule_info* info);
/* BN batch statistics -> scale/shift for bn_act_apply, saved mean/invstd for the backward, moving-stat update
 * (biased variance normalises, unbiased variance feeds the moving average; moving_* nullable). */
int yb_bn_finalize(const float* sum, const float* sqsum, long count, int c, const float* gamma, const float* beta,
                   float eps, float decay, float* moving_mean, float* moving_var, float* scale, float* shift,
                   float* save_mean, float* save_invstd, void* stream);
/* out = leaky(z*scale+shift) (+res); z/res/out 16-bit [n*h*w, ld]; upsample2x stores every row to its 4 places. */
int yb_bn_act_apply(const void* z, long z_ld, const float* scale, const float* shift, const void* res, long res_ld,
                    void* out, long out_ld, int n, int h, int w, int c, int dtype, int leaky, int upsample2x,
                    void* stream);
/* yb_bn_finalize + yb_bn_act_apply in ONE launch (count = n*h*w; same arguments, bit-identical results): the training
 * forward of a BN conv (slim.batch_norm(is_training=True) + leaky_relu, reference model.py:35-41). */
int yb_bn_stats_act_apply(const void* z, long z_ld, const float* sum, const float* sqsum, const float* gamma,
                          const float* beta, float eps, float decay, float* moving_mean, float* moving_var,
                          float* scale, float* shift, float* save_mean, float* save_invstd, const void* res,
                          long res_ld, void* out, long out_ld, int n, int h, int w, int c, int dtype, int leaky,
                          int upsample2x, void* stream);
/* Host-only: the launch shape of the BN streaming kernels (yb_bn_act_apply, yb_bn_stats_act_apply, yb_bn_bwd_reduce,
 * yb_bn_bwd_apply) for `rows` = n*h*w rows of c channels on a device with sm_count SMs, with the current options
 * (YB_BN_CPT).  A thread owns cpt consecutive channels (cv = c / cpt channel vectors per row) of one of `lanes` =
 * 256 / cv row lanes and walks its rows r unrolled (rows lane, lane + lanes, ...); block b owns rows
 * [b * rows_per_block, min((b + 1) * rows_per_block, rows)), rows_per_block a multiple of lanes chosen so that
 * grid <= sm_count * blocks_per_sm (one wave of co-resident blocks). */
typedef struct yb_bn_schedule_info {
  int cpt;             /* channels per thread: 8, or 4 (YB_BN_CPT=4, 32 <= c <= 1024) */
  int r;               /* rows in flight per thread (unroll)                           */
  int blocks_per_sm;
  int cv;              /* channel vectors per row                                      */
  int lanes;           /* row lanes per 256-thread block                               */
  long rows_per_block;
  int grid;
} yb_bn_schedule_info;
int yb_bn_schedule(long rows, int c, int sm_count, yb_bn_schedule_info* info);
/* dgamma/dbeta (fp32 [c], overwritten) from dA (gradient w.r.t. the layer output; upsample2x: summed over the
 * 4 copies) and the saved z.  workspace: NULL (atomic accumulation) or yb_bn_bwd_reduce_workspace_bytes() bytes,
 * zero-initialised once (two-stage deterministic reduction, no same-address atomics). */
int yb_bn_bwd_reduce_workspace_bytes(size_t* bytes);
int yb_bn_bwd_reduce(const void* dA, long dA_ld, const void* z, long z_ld, const float* scale, const float* shift,
                     const float* save_mean, const float* save_invstd, int n, int h, int w, int c, int dtype,
                     int leaky, int upsample2x, float* dgamma, float* dbeta, void* workspace, void* stream);
/* dz = gamma*invstd*(dact - dbeta/M - zhat*dgamma/M); dilate2x stores row (p,q) at (2p,2q) of [n,2h,2w,dz_ld]. */
int yb_bn_bwd_apply(const void* dA, long dA_ld, const void* z, long z_ld, const float* gamma, const float* scale,
                    const float* shift, const float* save_mean, const float* save_invstd, const float* dgamma,
                    const float* dbeta, int n, int h, int w, int c, int dtype, int leaky, int upsample2x,
                    int dilate2x, void* dz, long dz_ld, void* stream);
/* out[c] (fp32, overwritten) = column sums of x [rows, ld] (bias gradient of the detection convs). */
int yb_col_sum(const void* x, long ld, long rows, int c, int dtype, float* out, void* stream);
/* column sums and sums of squares (BN batch statistics of the stem's raw output). */
int yb_col_stats(const void* x, long ld, long rows, int c, int dtype, float* sum, float* sqsum, void* stream);

/* ---------------------------------------------------------------------------------
 * Decode  (replaces the ~40 elementwise TF ops of model.py:82-190 and the caller's
 * pred_scores = pred_confs * pred_probs, test_single_image.py:55)
 * --------------------------------------------------------------------------------- */
/* reorg_layer (model.py:82-137) for one scale.  anchors3x2: host float[6] (w,h) pixels.
 * xy_offset [gh,gw,1,2], boxes [n,gh,gw,3,4] (cx,cy,w,h px), conf_logits [n,gh,gw,3,1],
 * prob_logits [n,gh,gw,3,C]; any output may be NULL. */
int yb_reorg_layer(const float* feature_map, int n, int gh, int gw, int img_h, int img_w, int class_num,
                   const float* anchors3x2, float* xy_offset, float* boxes, float* conf_logits,
                   float* prob_logits, void* stream);
/* predict (model.py:140-190) over the three scales (/32,/16,/8).  anchors9x2: host float[18].
 * boxes [n,B,4] xyxy, confs [n,B,1] (nullable), probs [n,B,C] (nullable), scores [n,B,C] = conf*prob (nullable),
 * B = 3*(h/32*w/32 + h/16*w/16 + h/8*w/8). */
int yb_predict(const float* fm1, const float* fm2, const float* fm3, int n, int img_h, int img_w, int class_num,
               const float* anchors9x2, float* boxes, float* confs, float* probs, float* scores, void* stream);

/* ---------------------------------------------------------------------------------
 * NMS  (replaces utils/nms_utils.py:8-48: greater_equal + boolean_mask x2 +
 * tf.image.non_max_suppression + gather x3 per class + concat x3)
 * --------------------------------------------------------------------------------- */
int yb_nms_workspace_bytes(int n_images, int num_boxes, int num_classes, int max_boxes, size_t* bytes);
/* Per image and class: keep score >= score_thresh, greedy NMS (IoU > iou_thresh suppresses; TF CPU-kernel
 * arithmetic), at most max_boxes per class; classes concatenated ascending, descending score inside a class.
 *   boxes [n,B,4] xyxy, scores [n,B,C]
 *   out_boxes [n, C*max_boxes, 4], out_scores / out_labels / out_indices [n, C*max_boxes]
 *   out_indices = index of the kept box in the ORIGINAL [B] axis (not exposed by the reference)
 *   out_counts [n] (device int32) = K of each image. */
int yb_nms(const float* boxes, const float* scores, int n_images, int num_boxes, int num_classes, int max_boxes,
           float score_thresh, float iou_thresh, void* workspace, size_t workspace_bytes, float* out_boxes,
           float* out_scores, int32_t* out_labels, int32_t* out_indices, int32_t* out_counts, void* stream);

/* ---------------------------------------------------------------------------------
 * PASCAL-VOC evaluation  (replaces utils/eval_utils.py:311-423 voc_ap / voc_eval, called per class by
 * eval.py:114-137 and train.py's validation): detections of a whole validation set are matched batch by batch
 * into a caller-owned pool of 64-bit records, then sorted and reduced to per-class (npos, nd, rec, prec, ap).
 * --------------------------------------------------------------------------------- */
/* ground-truth boxes per image that yb_voc_match accepts (vmax) */
enum { YB_VOC_MAX_GT = 1024 };
/* Match one batch of NMS output to its ground truth and append one record per detection at pool[pool_offset + ...].
 *   out_boxes [n, cap, 4] float32 xyxy, out_scores / out_labels [n, cap], counts [n] int32: yb_nms / yb_net_detect
 *   output (classes ascending, score descending inside a class; entries past counts[i], clamped to [0, cap], ignored)
 *   gt_boxes [n, vmax, 4] float64 xyxy, gt_labels [n, vmax] int32, gt_counts [n] int32 (clamped to [0, vmax]);
 *   labels outside [0, num_classes) belong to no class.  vmax <= YB_VOC_MAX_GT.
 *   Image i's records go to pool_offset + counts[0] + ... + counts[i-1] onward (same order as out_*); the caller keeps
 *   pool_offset + sum(counts) <= pool_capacity (records past the capacity are dropped).
 *   class_counts [num_classes][2] uint64 (npos, nd) is ACCUMULATED into: zero it when a new evaluation starts.
 * The rule is voc_eval's: a detection is a TP iff the first gt box of its class with the highest '+1 pixel' IoU
 * (float64; the detection's own area in float32) has IoU > iou_thresh and no higher-scored detection of the same
 * (image, class) took it. */
int yb_voc_match(const float* out_boxes, const float* out_scores, const int32_t* out_labels, const int32_t* counts,
                 int n, int cap, const double* gt_boxes, const int32_t* gt_labels, const int32_t* gt_counts, int vmax,
                 int num_classes, double iou_thresh, uint64_t* pool, long pool_offset, long pool_capacity,
                 uint64_t* class_counts, void* stream);
/* out [num_classes][5] float64 = voc_eval(...) of every class over the first pool_size records: (npos, nd, rec, prec,
 * ap), (1e-6, 1e-6, 0, 0, 0) for a class without detections.  Detections are ranked by descending score, ties in pool
 * order (a stable sort).  use_07_metric: 11-point AP (bit-exact), else the area under the precision envelope (summed in
 * a different order than numpy: equal within 1e-12).  The pool is not modified.  num_classes <= 65535,
 * pool_size < 2^31. */
int yb_voc_ap_workspace_bytes(long pool_size, int num_classes, size_t* bytes);
int yb_voc_ap(const uint64_t* pool, long pool_size, const uint64_t* class_counts, int num_classes, int use_07_metric,
              void* workspace, size_t workspace_bytes, double* out, void* stream);

/* ---------------------------------------------------------------------------------
 * k-means anchors  (replaces get_kmeans.py:32-41 avg_iou and :59-93 kmeans, run by `python get_kmeans.py`,
 * README.md:121-133): one Lloyd iteration is yb_kmeans_assign, a [k + 1] read on the host, then yb_kmeans_median.
 * boxes [rows, 2] float64 (w, h), 16-byte aligned, every value finite and > 0 (the caller checks this: the median
 * orders values by their bits); clusters [k, 2] float64.  1 <= k <= YB_KMEANS_MAX_K, k <= rows < 2^31.
 * All three share one workspace of yb_kmeans_workspace_bytes(rows, k) bytes (too small: YB_ERR_WORKSPACE).
 * --------------------------------------------------------------------------------- */
enum { YB_KMEANS_MAX_K = 32 };
int yb_kmeans_workspace_bytes(long rows, int k, size_t* bytes);
/* get_kmeans.py:80-83: assign[i] = np.argmin over c of 1 - iou(boxes[i], clusters) (float64 in the reference's
 * operation order, first minimum).  result [k + 1] int32 is overwritten: result[c] = boxes assigned to c,
 * result[k] = boxes whose assignment differs from last_assign (get_kmeans.py:85 stops when it is 0).
 * last_assign may be assign itself. */
int yb_kmeans_assign(const double* boxes, long rows, const double* clusters, int k, const int32_t* last_assign,
                     int32_t* assign, int32_t* result, void* workspace, size_t workspace_bytes, void* stream);
/* get_kmeans.py:88-89: clusters_out[c] = np.median(boxes[assign == c], axis=0), bit for bit (a radix select of ranks
 * (m-1)/2 and m/2 per column; an even count averages them as numpy does).  counts [k] = result[0..k) of the
 * yb_kmeans_assign that wrote assign.  A cluster with count 0 gets NaN, as np.median of nothing does. */
int yb_kmeans_median(const double* boxes, long rows, const int32_t* assign, const int32_t* counts, int k,
                     double* clusters_out, void* workspace, size_t workspace_bytes, void* stream);
/* get_kmeans.py:32-41: out (one device double) = np.mean of every box's max IoU over the clusters, bit for bit: the
 * same pairwise summation tree numpy uses, then / rows.  Needs rows >= 1 only, and a workspace of
 * yb_kmeans_workspace_bytes(rows, 1) bytes whatever k is. */
int yb_kmeans_avg_iou(const double* boxes, long rows, const double* clusters, int k, double* out, void* workspace,
                      size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------
 * JPEG decode  (replaces cv2.imread(pic_path) at utils/data_utils.py:130 and test_single_image.py:38): baseline
 * JPEG files -> uint8 BGR pixels equal to cv2.imread of OpenCV 4.13 (IMREAD_COLOR, EXIF orientation applied), in
 * the yb_resize_batch / PackedImages layout.  Supported: SOF0 / SOF1, 8-bit Huffman, 1 component (grey, replicated
 * to BGR) or 3 components YCbCr, luma sampling 1x1, 2x1, 1x2 or 2x2 with chroma 1x1, one interleaved scan, restart
 * intervals, EXIF orientation 1-8.  Everything else (also an SOS that lists the components in another order than SOF,
 * or a stream past 2^32 bits once each restart segment is padded to a subsequence) is YB_ERR_UNSUPPORTED with the
 * reason; a malformed header is
 * YB_ERR_INVALID_ARGUMENT.  Batch calls prefix the reason with "image <index>: ".
 * --------------------------------------------------------------------------------- */
typedef struct yb_jpeg_info {
  int height, width;           /* of the decoded (EXIF-oriented) image                           */
  int src_height, src_width;   /* as stored in SOF                                               */
  int components;              /* 1 or 3                                                         */
  int h_samp, v_samp;          /* luma sampling factors (chroma is 1x1); 1x1 for grey           */
  int restart_interval;        /* MCUs per restart interval, 0 = none                            */
  int orientation;             /* EXIF orientation 1-8 (1 without an Exif block)                 */
  int mode;                    /* 0 baseline (SOF0), 1 extended sequential Huffman (SOF1)        */
} yb_jpeg_info;
/* per-image decode status (int32, bits may combine); the image's pixels are unspecified when it is nonzero,
 * libjpeg would warn and fill grey.  Only that image's slot is written. */
enum {
  YB_JPEG_OK = 0,
  YB_JPEG_BAD_MARKER = 1,   /* a marker other than RSTn / EOI inside the entropy-coded data             */
  YB_JPEG_BAD_RST = 2,      /* RST markers out of sequence or more than the restart interval implies    */
  YB_JPEG_BAD_CODE = 4,     /* a Huffman code no table holds (the segment's decode stops there)         */
  YB_JPEG_BAD_INDEX = 8,    /* a coefficient index past 63 (likewise)                                   */
  YB_JPEG_TRUNCATED = 16    /* data (or restart segments) end before the last MCU                       */
};
/* host only: one file's header. */
int yb_jpeg_parse(const void* data, size_t bytes, yb_jpeg_info* info);
/* host only: the blob of n files (data[i], bytes[i]) that is the batch's one H2D copy: descriptors, quantisation
 * and Huffman decode tables, compressed bytes.  It records the subsequence size of the Huffman decode
 * (YB_JPEG_SUBSEQ_BITS) at pack time.  desc_host (optional) receives the int64 [n, 4] output table (pixel byte
 * offset, height, width, row pitch), each image 16-byte aligned as PackedImages packs them. */
int yb_jpeg_pack_bytes(const void* const* data, const size_t* bytes, int n, size_t* blob_bytes);
int yb_jpeg_pack(const void* const* data, const size_t* bytes, int n, void* host_blob, size_t blob_bytes,
                 int64_t* desc_host);
/* host only: workspace bytes of yb_jpeg_decode for this blob (destuffed streams, sync records, coefficient blocks,
 * component planes) and the pixel bytes out_pixels must hold (optional). */
int yb_jpeg_workspace_bytes(const void* host_blob, int n, size_t* bytes, size_t* pixel_bytes);
/* dev_blob: the device copy of host_blob (16-byte aligned).  Writes out_pixels and out_desc (int64 [n, 4], the
 * table yb_jpeg_pack returns) and status int32 [n].  Six launches for the whole batch, no host synchronisation. */
int yb_jpeg_decode(const void* dev_blob, const void* host_blob, int n, uint8_t* out_pixels, int64_t* out_desc,
                   int32_t* status, void* workspace, size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------
 * JPEG encode  (replaces cv2.imwrite / cv2.imencode('.jpg'), test_single_image.py:85): uint8 BGR or grey images on
 * the device -> baseline JPEG files equal byte for byte to cv2.imencode of OpenCV 4.13 (libjpeg-turbo 3.1) with the
 * same IMWRITE_JPEG_QUALITY, _SAMPLING_FACTOR, _RST_INTERVAL, _LUMA_QUALITY and _CHROMA_QUALITY.  Standard Huffman
 * tables, one interleaved scan (one component for grey).  A bad image description is YB_ERR_INVALID_ARGUMENT with
 * the reason; batch calls prefix it with "image <index>: ".
 * --------------------------------------------------------------------------------- */
enum {   /* sampling: OpenCV's IMWRITE_JPEG_SAMPLING_FACTOR_* values (luma h, v; chroma 1x1) */
  YB_JPEG_SAMPLING_411 = 0x411111,
  YB_JPEG_SAMPLING_420 = 0x221111,
  YB_JPEG_SAMPLING_422 = 0x211111,
  YB_JPEG_SAMPLING_440 = 0x121111,
  YB_JPEG_SAMPLING_444 = 0x111111
};
typedef struct yb_jpeg_enc_image {
  const void* pixels;          /* device address of row 0 (not read by the host-only calls)                    */
  int64_t pitch;               /* bytes from one row to the next, >= width * channels                          */
  int height, width;           /* 1..65535                                                                     */
  int channels;                /* 3: BGR (three-component YCbCr file), 1: grey (one-component file)            */
  int quality;                 /* IMWRITE_JPEG_QUALITY, clamped to 0..100 as OpenCV does                       */
  int luma_quality;            /* IMWRITE_JPEG_LUMA_QUALITY, < 0: not given                                    */
  int chroma_quality;          /* IMWRITE_JPEG_CHROMA_QUALITY, < 0: not given                                  */
  int sampling;                /* YB_JPEG_SAMPLING_*; grey ignores it                                          */
  int restart_interval;        /* IMWRITE_JPEG_RST_INTERVAL in MCUs, clamped to 0..65535; 0: none              */
} yb_jpeg_enc_image;
/* host only: the file's bytes up to and including SOS.  out NULL (or capacity too small: YB_ERR_WORKSPACE) only
 * reports the length in *bytes. */
int yb_jpeg_enc_header(const yb_jpeg_enc_image* image, uint8_t* out, size_t capacity, size_t* bytes);
/* host only: the blob of n images that is the batch's one H2D copy: image geometry, quantisation reciprocals,
 * Huffman code tables and headers. */
int yb_jpeg_enc_pack_bytes(const yb_jpeg_enc_image* images, int n, size_t* blob_bytes);
int yb_jpeg_enc_pack(const yb_jpeg_enc_image* images, int n, void* host_blob, size_t blob_bytes);
/* host only: workspace bytes of yb_jpeg_enc_encode for this blob and the output capacity out must have (an upper
 * bound on the n files together). */
int yb_jpeg_enc_workspace_bytes(const void* host_blob, int n, size_t* workspace_bytes, size_t* out_bytes);
/* dev_blob: the device copy of host_blob (16-byte aligned).  Writes the n files back to back from out[0] and
 * out_desc int64 [n, 2] = (byte offset, length).  Eight launches for the whole batch, no host synchronisation. */
int yb_jpeg_enc_encode(const void* dev_blob, const void* host_blob, int n, uint8_t* out, size_t out_bytes,
                       int64_t* out_desc, void* workspace, size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------
 * Detection drawing  (replaces utils/plot_utils.py plot_one_box and the loop of test_single_image.py:81-83 /
 * video_test.py:91): cv2.rectangle + filled label box + cv2.putText(FONT_HERSHEY_SIMPLEX, LINE_AA) per detection,
 * in order, equal to OpenCV 4.13's pixels, at every line thickness.
 * --------------------------------------------------------------------------------- */
enum { YB_PLOT_SUFFIX_MAX = 48 };            /* longest score suffix ", -<39 digits>.dd%" */
enum { YB_PLOT_BAD_LABEL = 1, YB_PLOT_BAD_BOX = 2 };
typedef struct yb_plot_layout {
  int length;                  /* label characters (FONT_HERSHEY_SIMPLEX codes ' ' .. '~') written to text     */
  int thickness;               /* font thickness max(tl - 1, 1)                                                */
  int text_w, text_h;          /* cv2.getTextSize(text, 0, tl / 3, thickness)[0]                               */
  int rect_x1, rect_y1;        /* the filled label rectangle runs from (x0, y0) to here                        */
  int org_x, org_y;            /* putText origin                                                               */
} yb_plot_layout;
/* host only: the label of one detection at corner (x0, y0): name (UTF-8, 0..255 bytes, each byte outside
 * ' ' .. '~' drawn as '?'), then with_score ? ", {:.2f}%" of the float32 score * 100 : nothing.  text needs
 * name_len + YB_PLOT_SUFFIX_MAX bytes.  The device computes every label with this same function. */
int yb_plot_label_layout(const unsigned char* name, int name_len, int with_score, float score, int tl, int x0,
                         int y0, unsigned char* text, yb_plot_layout* layout);
/* host only: bytes of the blob yb_plot_pack writes (the batch's one H2D copy), names_bytes the class names' total */
int yb_plot_workspace_bytes(int n, int classes, size_t names_bytes, size_t* bytes);
/* host only: tl [n] line thickness per image (0..1023), colors [classes, 3] (saturated
 * to 0..255, channel order of the image), names the class names back to back with name_len [classes] bytes each
 * (-1: no label, as plot_one_box(label=None)); with_score appends the score suffix to every label. */
int yb_plot_pack(const int* tl, int n, const int* colors, const unsigned char* names, const int* name_len,
                 int classes, int with_score, void* host_blob, size_t bytes);
/* Draws in place into data, the PackedImages layout (int64 [n, 4] descriptors (offset, h, w, pitch), then the
 * uint8 BGR pixels); max_h / max_w bound the images' sizes.  boxes [n, slots, 4] f32 (x0, y0, x1, y1), scores
 * [n, slots] f32 (may be NULL without the score suffix), labels [n, slots] i32 and counts [n] i32: detections
 * 0 .. counts[i] - 1 of image i are drawn in order.  Coordinates are truncated toward zero like int(); they are
 * first clamped to +-2^24, which changes no pixel of an image up to 65535 pixels a side.  A detection with a label
 * outside [0, classes) or a non-finite coordinate is skipped; status int32 [n, 2] gets (YB_PLOT_BAD_* flags, first
 * bad slot or -1).  One launch, no host synchronisation. */
int yb_plot_boxes(void* data, int n, int max_h, int max_w, const float* boxes, const float* scores,
                  const int* labels, const int* counts, int slots, const void* dev_blob, int* status, void* stream);

/* ---------------------------------------------------------------------------------
 * Loss  (replaces model.py:192-304 loss_layer, :307-345 box_iou, :348-365 compute_loss and
 * the part of TF autodiff (train.py:112) that differentiates them)
 * --------------------------------------------------------------------------------- */
int yb_loss_workspace_bytes(int n, int gh, int gw, size_t* bytes);
/* One scale.  feature_map [n,gh,gw,3*(5+C)] f32 logits, y_true [n,gh,gw,3,5+C+1] f32 (utils/data_utils.py:51-115
 * format: cx,cy,w,h px | obj | one-hot | mix-up weight), anchors3x2 host float[6].
 * loss4 (device double[4]: xy, wh, conf, class) is ACCUMULATED into (zero it first; every term already
 * carries the 1/N of model.py:276-302, N = 1/inv_batch).
 * dfm (nullable) receives d(total)/d(feature_map): dfm_dtype YB_F32 -> same layout as feature_map;
 * YB_F16/YB_BF16 -> [n*gh*gw, dfm_ld] rows (dfm_ld >= 3*(5+C), padding columns zeroed) for the backward GEMMs. */
/* loss_scale (> 0; 1 = off) multiplies the stored gradient only (not the loss values): the fp16 backward chain
 * needs it to keep small gradients above the subnormal range; the optimizer divides it out again
 * (yb_optimizer.grad_scale) and skips a step whose gradient is non-finite. */
int yb_loss_layer(const float* feature_map, const float* y_true, int n, int gh, int gw, int img_h, int img_w,
                  int class_num, const float* anchors3x2, int use_label_smooth, int use_focal_loss,
                  float inv_batch, float loss_scale, void* workspace, size_t workspace_bytes, double* loss4,
                  void* dfm, int dfm_dtype, int dfm_ld, void* stream);
/* out5 (device float[5]) = [total, xy, wh, conf, class] (model.py:364-365). */
int yb_loss_finalize(const double* loss4, float* out5, void* stream);
/* box_iou (model.py:307-345): pred_boxes [P,4], true_boxes [V,4] (cx,cy,w,h) -> iou [P,V]. */
int yb_box_iou(const float* pred_boxes, const float* true_boxes, long num_pred, int num_true, float* iou,
               void* stream);

/* ---------------------------------------------------------------------------------
 * Network plan: the 75-conv Darknet-53 + YOLOv3 head of model.py:30-80 for a fixed
 * (batch, H, W, dtype).  Holds tensor maps and the layer schedule; buffers are the
 * caller's: one activation arena and one parameter arena.
 * --------------------------------------------------------------------------------- */
typedef struct yb_net yb_net;

typedef struct yb_layer_info {
  int index;          /* creation order == TF variable order == darknet .weights order  */
  int cin, cout, ksize, stride;
  int has_bn;         /* 0 for the three detection convs (bias, linear)                  */
  int in_h, in_w, out_h, out_w;
  int is_head;        /* 1: under yolov3_head, 0: darknet53_body                        */
  int scope_index;    /* k of "Conv_k" inside its variable scope                        */
  int upsample2x;     /* 1: output is stored 2x nearest-neighbour upsampled (model.py:61,71) */
} yb_layer_info;

int yb_net_create(yb_net** net, int class_num, int n, int h, int w, int dtype, int training);
int yb_net_destroy(yb_net* net);
int yb_net_num_layers(const yb_net* net);
int yb_net_layer_info(const yb_net* net, int layer, yb_layer_info* info);
/* Host-only unless sm_count == 0: the kernel, multicast-cluster shape and persistent grid the forward of a plan
 * (yb_net_forward / yb_net_detect, current options) launches for `layer`.  sm_count > 0: a device with that many SMs,
 * max_clusters = sm_count / (cluster_m * cluster_n); sm_count == 0: the current device, max_clusters from
 * cudaOccupancyMaxActiveClusters for the kernel.  igemm = 0: the layer runs another kernel, named by `kernel`; of the
 * other fields only residual and res_smem are then set.  The detection heads are reported as yb_net_forward runs them
 * (unfused); det_block_n gives the tile width of their fused-decode launch in yb_net_detect.
 * kernel (every layer, layer 0 included):
 *   YB_LAYER_IGEMM       the implicit-GEMM conv (igemm = 1)
 *   YB_LAYER_HALO        the halo-tile kernel (Cin = 32 layers by default; YB_HALO=0: none, YB_HALO=1: wherever it applies)
 *   YB_LAYER_FUSED_STEM  layers 0 and 1: the stem is computed inside Conv_1's halo launch, layer 0's output is never
 *                        written (the default; YB_STEM_FUSE=0 or YB_HALO=0 turn it off)
 *   YB_LAYER_STEM        layer 0 as its own launch: the mma.sync stem, or the CUDA-core stem under YB_THIN=0
 *   YB_LAYER_THIN        the mma.sync halo-tile kernel of the Cin = 32 3x3 convs (YB_THIN=2) */
enum { YB_LAYER_IGEMM = 1, YB_LAYER_HALO = 2, YB_LAYER_FUSED_STEM = 3, YB_LAYER_STEM = 4, YB_LAYER_THIN = 5 };
typedef struct yb_layer_schedule_info {
  int igemm;         /* 1: the implicit-GEMM conv                                                  */
  int pingpong;      /* 1: ping-pong schedule, 0: cooperative                                       */
  int cluster_m;     /* CTAs of a cluster along M (each a different m-tile)                         */
  int cluster_n;     /* CTAs of a cluster along N (1 | 2; 1 under the cooperative schedule)         */
  int block_m, block_n;
  int num_m_tiles, num_n_tiles;
  int units;         /* work units: ceil(num_m_tiles / cluster_m) x num_n_tiles / cluster_n         */
  int max_clusters;  /* most clusters resident at once                                              */
  int grid;          /* CTAs launched: a multiple of cluster_m x cluster_n, <= max_clusters of them */
  int residual;      /* 1: the layer adds a shortcut (also reported for the halo-kernel layers)     */
  int res_smem;      /* 1: the shortcut tile is TMA-prefetched into shared memory during the main   */
                     /*    loop (YB_CONV_RES); 0: the epilogue reads it from global memory          */
  int kernel;        /* YB_LAYER_*: what the forward launches for this layer (above)                */
  int epi_tma;       /* 1: the TMA-store epilogue (YB_CONV_EPI); 0: the staged or register epilogue  */
  int det_block_n;   /* detection heads: columns of the one n-tile of the fused-decode launch, the   */
                     /*    narrowest of 64, 128, 256 that holds 3 (5 + C); 0: none (C > 80), or not a head */
} yb_layer_schedule_info;
int yb_net_layer_schedule(const yb_net* net, int layer, int sm_count, yb_layer_schedule_info* info);
int yb_net_arena_bytes(const yb_net* net, size_t* activation_bytes, size_t* param_bytes);
/* Bind caller-owned arenas (256-byte aligned).  Must be called before set_params/forward.  The PARAMETER arena layout
 * depends only on (class_num, dtype, training): plans of different batch / image sizes may share one parameter arena
 * (master weights, 16-bit copies, folded BN, optimizer slots) — this is how one model serves multi-scale training
 * (train.py:47-49 multi_scale_train) with a single set of weights and a single optimizer state.  Binding fills
 * constants and this plan's activation-arena scratch on `stream`; it never touches weights or optimizer slots. */
int yb_net_bind(yb_net* net, void* activation_arena, size_t activation_bytes, void* param_arena,
                size_t param_bytes, void* stream);
/* Re-fold every BN layer's (gamma, beta, moving mean, moving variance) into the inference scale/shift (needed after
 * training steps made through ANOTHER plan that shares the parameter arena; a plan refolds by itself after its own). */
int yb_net_refold_bn(yb_net* net, void* stream);
/* Upload one conv's parameters (device float32 pointers).  BN layers: gamma,beta,mean,var (bias NULL);
 * detection convs: bias (others NULL).  Repacks/folds on `stream`. */
int yb_net_set_conv_params(yb_net* net, int layer, const float* w, int layout, const float* gamma,
                           const float* beta, const float* mean, const float* var, const float* bias,
                           void* stream);
/* forward (model.py:30-80), inference mode: images float32 [n,h,w,3] -> fm1 [n,h/32,w/32,D],
 * fm2 [n,h/16,w/16,D], fm3 [n,h/8,w/8,D] float32, D = 3*(5+class_num). */
int yb_net_forward(yb_net* net, const float* images, float* fm1, float* fm2, float* fm3, void* stream);
/* The whole detection pipeline of test_single_image.py:50-57 in one call:
 *   forward (model.py:30-80) -> predict (model.py:140-190) -> pred_scores = confs * probs (test_single_image.py:55)
 *   -> gpu_nms per image (utils/nms_utils.py:8-48; max_boxes per class, score >= score_thresh, IoU > iou_thresh suppresses).
 * The decode and the score filter run INSIDE the epilogues of the three detection-head convs (fp32 accumulators ->
 * boxes + per-(image, class) candidate lists); the feature maps and the [n, B, C] score tensor are never written.
 * Results are bit-identical to yb_net_forward + yb_predict + yb_nms.
 *   anchors9x2 host float[18] (w,h pixels, small -> large);  boxes [n, B, 4] float32 out: every decoded box
 *   (xmin,ymin,xmax,ymax), B = 3*(h/32*w/32 + h/16*w/16 + h/8*w/8);  workspace >= yb_net_detect_workspace_bytes;
 *   out_* as yb_nms (fixed shape [n, class_num*max_boxes(,4)], out_counts [n]).
 * yb_net_detect_supported: 1 when the plan is bound and its class count has fused heads (1 to 80 classes, every
 * dtype), else 0 — callers then use the three separate calls. */
int yb_net_detect_supported(const yb_net* net);
int yb_net_detect_workspace_bytes(const yb_net* net, int max_boxes, size_t* bytes);
int yb_net_detect(yb_net* net, const float* images, const float* anchors9x2, int max_boxes, float score_thresh,
                  float iou_thresh, void* workspace, size_t workspace_bytes, float* boxes, float* out_boxes,
                  float* out_scores, int32_t* out_labels, int32_t* out_indices, int32_t* out_counts, void* stream);
/* yb_net_detect split for benchmarks that bracket its parts with their own events: phases is a bit mask,
 * 1 = candidate-list reset + stem (layer 0), 2 = the 74 tensor-core convs (decode fused into the heads), 4 = NMS
 * selection + gather.  yb_net_detect == phases 7. */
int yb_net_detect_phases(yb_net* net, const float* images, const float* anchors9x2, int max_boxes, float score_thresh,
                         float iou_thresh, void* workspace, size_t workspace_bytes, float* boxes, float* out_boxes,
                         float* out_scores, int32_t* out_labels, int32_t* out_indices, int32_t* out_counts, int phases,
                         void* stream);
/* Same, restricted to layers [first, last] (creation order) — lets a benchmark bracket the CUDA-core stem
 * (layer 0) and the tensor-core convs (1..74) with its own events. */
int yb_net_forward_layers(yb_net* net, const float* images, float* fm1, float* fm2, float* fm3, int first,
                          int last, void* stream);
/* ---- training plan (yb_net_create(..., training=1)); one reference training step (train.py:105-115) is
 *      yb_net_train_fwd_bwd -> [all-reduce of yb_net_grad_buffer across ranks] -> yb_net_train_update ---- */
/* forward with BN batch statistics (updating the moving statistics with `bn_decay`, train.py:108-109) ->
 * compute_loss (model.py:348-365; loss4 = device double[4] xy,wh,conf,class, overwritten) -> backward into the
 * flat gradient buffer (data term only).  YB_TRAIN_FORWARD_ONLY stops after the forward (y_true*, loss4 may be NULL).
 * y_true_k: [n, g_k, g_k, 3, 5+C+1] float32 for the /32, /16, /8 maps; anchors9x2 host float[18].
 * fm1..3 nullable (then the arena-owned float32 outputs are used). */
/* flags: YB_TRAIN_FORWARD_ONLY stops after the forward; YB_TRAIN_BN_FROZEN normalises with the moving statistics
 * (forward(is_training=False) inside the training graph: fine-tuning with frozen BN; statistics are constants of the
 * backward pass and are not updated) — per-image results then do not depend on the rest of the batch, which is what
 * makes an N-rank data-parallel step bit-comparable with a 1-rank step on the concatenated batch. */
enum { YB_TRAIN_FORWARD_ONLY = 1, YB_TRAIN_BN_FROZEN = 2, YB_TRAIN_NO_BACKWARD = 4 };
int yb_net_train_fwd_bwd(yb_net* net, const float* images, const float* y_true_1, const float* y_true_2,
                         const float* y_true_3, const float* anchors9x2, int use_label_smooth, int use_focal_loss,
                         float bn_decay, float loss_scale, float* fm1, float* fm2, float* fm3, double* loss4,
                         int flags, void* stream);
/* Bucketed data parallelism (SURVEY.md 8e): yb_net_train_fwd_bwd(..., flags | YB_TRAIN_NO_BACKWARD) stops after the
 * loss; yb_net_train_backward then runs the backward of layers last_layer .. first_layer (descending, same flags), and
 * yb_net_grad_range returns the contiguous slice of the flat gradient those layers own — the caller issues the
 * all-reduce of a finished bucket (detection heads first) while the next bucket's backward is running. */
int yb_net_train_backward(yb_net* net, const float* images, int first_layer, int last_layer, int flags, void* stream);
int yb_net_grad_range(yb_net* net, int first_layer, int last_layer, float** ptr, size_t* count);
/* ---- synchronised batch norm for data-parallel training: the step as per-layer calls with exchange points ----
 * Each layer runs in two phases.  YB_PHASE_LOCAL computes per-replica sums: forward, the conv and its batch sums
 * Σz / Σz² (layer 0 also zeroes the per-step sums and, unless YB_TRAIN_FORWARD_ONLY, the flat gradient); backward,
 * the BN gradient sums Σdact·ẑ / Σdact.  YB_PHASE_GLOBAL consumes them: forward, statistics -> scale / shift, the
 * moving-statistics update and the activation; backward, dz, the weight gradient (on a side stream) and the input
 * gradient.  Between the two phases of a BN layer the caller sums the layer's exchange slab (yb_net_bn_exchange_buffer)
 * across the ranks in place.  A detection conv (no BN) has nothing to exchange: its forward runs in LOCAL, its bias
 * gradient in backward LOCAL.
 * Order of one step: forward_layer(0, LOCAL), (0, GLOBAL), ... (74, GLOBAL); train_loss; backward_layer(74, LOCAL),
 * (74, GLOBAL), ... (0, GLOBAL); then yb_net_train_join and yb_net_train_update.  A call out of this order fails with
 * YB_ERR_INVALID_ARGUMENT before any device work; forward_layer(0, LOCAL) always starts a new step.
 * bn_replicas (>= 1, the same for every call of a step) multiplies the rows the statistics cover:
 * M = bn_replicas * n * out_h * out_w, in the mean / variance, the backward and the unbiased-variance factor of the
 * moving-statistics update.  Every rank must therefore run the same n, H and W in a step.  With bn_replicas = 1 and
 * no exchange the calls compute what yb_net_train_fwd_bwd computes.  The flat gradient holds the LOCAL dgamma / dbeta
 * and rank-local weight gradients whose all-reduce times 1/world is the gradient of the concatenated batch. */
enum { YB_PHASE_LOCAL = 0, YB_PHASE_GLOBAL = 1 };
int yb_net_train_forward_layer(yb_net* net, const float* images, int layer, int phase, int bn_replicas, float bn_decay,
                               float* fm1, float* fm2, float* fm3, int flags, void* stream);
/* compute_loss of yb_net_train_fwd_bwd on the feature maps the forward wrote: zeroes loss4, then accumulates into it
 * and writes d(loss)/d(feature maps) for the backward. */
int yb_net_train_loss(yb_net* net, const float* y_true_1, const float* y_true_2, const float* y_true_3,
                      const float* anchors9x2, int use_label_smooth, int use_focal_loss, float loss_scale,
                      double* loss4, void* stream);
int yb_net_train_backward_layer(yb_net* net, const float* images, int layer, int phase, int bn_replicas, int flags,
                                void* stream);
/* makes `stream` wait for the weight-gradient side stream: call before all-reducing a finished gradient range and
 * after the last backward call. */
int yb_net_train_join(yb_net* net, void* stream);
/* BN layer `layer`'s exchange slab, 2 x cout_pad floats: forward [Σz | Σz²], backward [Σdact·ẑ | Σdact]. */
int yb_net_bn_exchange_buffer(yb_net* net, int layer, int backward, float** ptr, size_t* count);
/* Read-only view of BN layer `layer`'s coefficients from the last training forward, fp32 [cout] each (activation
 * arena): the mean it normalised with (the moving mean under YB_TRAIN_BN_FROZEN), invstd = rsqrtf(var + eps), and
 * scale = gamma * invstd, shift = beta - mean * scale, which the activation and the backward read.  Needs a bound
 * training plan and a layer with batch norm (YB_ERR_INVALID_ARGUMENT otherwise); a NULL output is skipped. */
int yb_net_bn_batch_stats(yb_net* net, int layer, float** mean, float** invstd, float** scale, float** shift);
/* the flat float32 gradient of all 222 trainable tensors (creation order: per conv w [OHWI], then gamma, beta
 * | bias; each padded to 4 floats) — the buffer a data-parallel wrapper all-reduces. */
int yb_net_grad_buffer(yb_net* net, float** ptr, size_t* count);
/* The optimizers of utils/misc_utils.py:151-161 (config_optimizer) with TensorFlow 1.x update rules. */
typedef enum yb_opt_kind {
  YB_OPT_SGD = 0,      /* GradientDescentOptimizer: w -= lr*g                                                    */
  YB_OPT_MOMENTUM = 1, /* MomentumOptimizer(momentum): v = m*v + g; w -= lr*v  (the reference's default)         */
  YB_OPT_RMSPROP = 2,  /* RMSPropOptimizer(decay, momentum, epsilon=1e-10): ms = d*ms + (1-d)g^2 (ms starts at 1);
                          mom = m*mom + lr*g/sqrt(ms+eps); w -= mom                                              */
  YB_OPT_ADAM = 3      /* AdamOptimizer(beta1=.9, beta2=.999, epsilon=1e-8): lr_t = lr*sqrt(1-b2^t)/(1-b1^t);
                          m = b1*m + (1-b1)g; v = b2*v + (1-b2)g^2; w -= lr_t*m/(sqrt(v)+eps)                    */
} yb_opt_kind;
typedef struct yb_optimizer {
  int kind;            /* yb_opt_kind                                                                            */
  float lr;            /* THIS step's learning rate: the host evaluates the schedule (utils/misc_utils.py:129-148,
                          warm-up train.py:93-99; Python: utils.misc_utils.config_learning_rate)                 */
  float grad_scale;    /* multiplies the raw gradient buffer: 1/world_size (data-parallel mean) x 1/loss_scale   */
  float momentum, decay, beta1, beta2, epsilon;
  float weight_decay;  /* slim.l2_regularizer on conv weights only (model.py:49, train.py:78)                    */
  float clip_norm;     /* per-tensor tf.clip_by_norm (train.py:113-114); <= 0: off                               */
} yb_optimizer;
/* g = grad_scale*grad + weight_decay*w (conv weights only); per-tensor clip_by_norm; the optimizer's rule on the fp32
 * master weights and its slots; refresh of the 16-bit compute copies and dgrad weights.  A step whose gradient holds
 * a non-finite value is skipped entirely (yb_net_opt_state: ctrl[2] counts skipped steps, ctrl[1] applied ones). */
int yb_net_train_update(yb_net* net, const yb_optimizer* opt, void* stream);
/* Zero the optimizer slots (rmsprop: mean-square slot = 1 like TF), the gradient buffer and the step counters.
 * Call once when a parameter arena starts training (or the optimizer changes); binding a plan never does this. */
int yb_net_train_reset_state(yb_net* net, int optimizer_kind, void* stream);
/* The optimizer slots: num_slots x count_per_slot floats laid out like the gradient buffer, and int ctrl[3] =
 * {non-finite flag of the running step, updates applied, steps skipped} (checkpoint save/restore of save_optimizer,
 * train.py:101-104,118-121). */
int yb_net_opt_state(yb_net* net, float** slots, size_t* count_per_slot, int* num_slots, int** ctrl);
/* Read-only view of the per-tensor squared norms the last yb_net_train_update computed and clipped with: float
 * sqnorm[count], the fp32 sum over a tensor's elements of (grad_scale*grad + weight_decay*w)^2 (0 for a tensor excluded
 * by yb_net_set_trainable).  count = 2 + 3 * 72 = 222: per layer in creation order, w, then gamma and beta (BN layers)
 * or bias (detection convs). */
int yb_net_opt_norms(yb_net* net, float** sqnorm, int* count);
/* train.py:81 update_part: exclude a conv (weights + gamma/beta | bias) from / include it in the update. */
int yb_net_set_trainable(yb_net* net, int layer, int trainable, void* stream);
/* Re-derive the dgrad weight layouts from the fp32 master weights (after the arena's weights were replaced). */
int yb_net_train_refresh_dgrad(yb_net* net, void* stream);
/* device pointers of one conv's float32 master parameters (w is OHWI [cout,k,k,cin]) / of its gradients. */
int yb_net_get_conv_params(yb_net* net, int layer, float** w_ohwi, float** gamma, float** beta, float** mean,
                           float** var, float** bias);
int yb_net_layer_grad(yb_net* net, int layer, float** dw, float** dgamma, float** dbeta, float** dbias);
/* training scratch of one layer (tests), 16-bit, h x w rows of row pitch ld:
 *   0  z: the raw conv output, [n, out_h, out_w, ld]
 *   1  dz: its gradient, [n, out_h, out_w, ld] (YB_DGRAD_S2=dilated stride-2 layers: zero-inserted at the input
 *      resolution); the detection heads' dz has ld = cout rounded up to 32, the pad columns zero
 *   2  dA: the gradient w.r.t. the layer output, [n, h, w, ld] (2x upsampled outputs: at the upsampled size)
 *   3  in: the layer's input activation, [n, in_h, in_w, ld] (a concat slice: ld is the concat buffer's)
 *   4  the dgrad weights (parameter arena): rows h = cin_pad x w = k * k taps, ld = k_cout (cout rounded up to 32);
 *      stride-1 layers hold the flip + transpose of the weights, stride-2 parity layers the four class matrices
 *   5  dX: the gradient w.r.t. the layer's input, the tensor its dgrad writes, [n, in_h, in_w, ld]
 *   6  w16: the 16-bit forward weights (parameter arena), h = cout_pad rows x w = 1 of ld = k * k * cin (OHWI)
 * Layer 0 (the stem) has no 3, 4, 5 or 6. */
int yb_net_train_buffer(yb_net* net, int layer, int which, void** ptr, int* ld, int* h, int* w);
/* device pointer + geometry of one layer's output activation (tests / debugging). */
int yb_net_layer_output(const yb_net* net, int layer, void** ptr, int* ld, int* dtype);
/* ---- calibrated fp8 inference plan: yb_net_create(..., YB_E4M3, training = 0) ----
 * Layers 0-3 (the stem, Conv_1, Conv_2, Conv_3) compute in fp16; Conv_3's output and every later non-head activation
 * buffer is e4m3 with one float32 scale per buffer; the heads write float32.  Weights of layers >= 4 are e4m3 with
 * per-output-channel scales (yb_pack_conv_weights_e4m3, applied by yb_net_set_conv_params), and the folded scale of
 * each such layer is (BN scale) x (input buffer scale) x (weight scale).  yb_net_set_fp8_amax takes one amax per layer
 * (host float[num_layers], e.g. yb_amax of the layer outputs of an fp16 plan over calibration images; entries of layers
 * whose output is not e4m3 are ignored): a buffer's scale is max(amax of the layers writing it) / 448 (1 if that is 0),
 * and the plan refolds.  Until it is called, forward / detect on the plan fail.  yb_net_fp8_layer_scales: the input,
 * residual and output buffer scales of one layer (host float[3]) and its device weight scales (NULL for layers 0-3). */
int yb_net_set_fp8_amax(yb_net* net, const float* amax, int count, void* stream);
int yb_net_fp8_layer_scales(const yb_net* net, int layer, float* in_res_out, float** w_scale);
/* number of kernels one yb_net_forward enqueues (for bench.py's gpu_launches). */
int yb_net_forward_launches(const yb_net* net);

#ifdef __cplusplus
}
#endif
#endif /* YOLOB200_H_ */
