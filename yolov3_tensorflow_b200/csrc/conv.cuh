// Shared between the wgmma conv files (conv_igemm.cu, conv_halo.cu, conv_wgrad.cu) and the network plan (net.cu,
// net_train.cu).
#pragma once
#include "common.cuh"
#include "decode.cuh"

namespace yb {

struct ConvParams {
  int M, P, Q;            // output pixels (n*P*Q), output height, width
  int cout;               // valid output channels
  int cin;                // input channels (K per filter tap)
  int ksize, stride, pad;
  int kh, kw;             // filter window (ksize x ksize for the forward convs; 1x1 .. 2x2 for the stride-2 dgrad classes)
  int scatter;            // 0, or 1 + 2a + b: output pixel (p, q) is stored at (2p + a, 2q + b) of a [n, 2P, 2Q] grid
  int im2col;             // 1: A via im2col TMA, 0: A via 2D tiled TMA
  int consumers;          // consumer warpgroups per CTA: 64 output rows each (1 | 2)
  int cluster;            // CTAs per cluster (1 | 2 | 4), both schedules: (cluster / cluster_n) x cluster_n m x n tiles,
                          // each CTA multicasting its slice of the A tile along N and of the B tile along M
  int cluster_n;          // CTAs of a cluster along N (1 | 2; conv_select gives the cooperative schedule 1)
  int epi_reg;            // 1: accumulator fragments stored straight from registers (no staging tile)
  int pingpong;           // 1: the two consumer warpgroups take whole tiles in turn (csrc/conv_igemm.cu)
  int ctas;               // > 0: the persistent grid is capped at this many CTAs (YB_CONV_CTAS; conv_grid)
  int num_m_tiles, num_n_tiles;
  const float* scale;     // [cout_pad]
  const float* shift;     // [cout_pad]
  void* out;
  long out_ld;
  const void* res;
  long res_ld;
  int out_fp32, leaky, upsample;
  float* stat_sum;        // nullable: BN batch statistics of the raw conv result
  float* stat_sqsum;
  DetParams det;          // det.on: decode + NMS candidate filter instead of the fp32 feature-map store (detection heads)
  // e4m3 only (1 otherwise): the residual buffer's scale (codes -> values) and 1 / the output buffer's scale
  float res_scale, out_inv_scale;
  int res_smem;           // 1: the ping-pong kernel TMA-prefetches the residual tile into shared memory (YB_CONV_RES)
  CUtensorMap tmR;        // res_smem: the residual as a [M, cout] matrix, 128-row x 64-channel 128B-swizzled boxes
  int epi_tma;            // 1: the epilogue stays in the accumulator layout and stores 16-bit boxes by TMA (YB_CONV_EPI)
  CUtensorMap tmO;        // epi_tma: the output as a [M, cout] matrix of pitch out_ld, 16-row x 64-channel 128B-swizzled boxes
  // The rest of the conv_igemm_kernel instantiation conv_select picks (consumers, pingpong, cluster, cluster_n,
  // res_smem and epi_tma above are the others); host only, after every field the kernel reads.
  int dtype;              // yb_dtype of the operands
  int block_n;            // output channels per tile
  int block_kb;           // bytes of one k-block row
  int det_e;              // > 0: the fused-decode head kernel for 5 + C = det_e columns per anchor
};

// One implicit-GEMM launch (host only): the operand tensor maps and the parameters they were encoded for.  The TMA
// boxes depend on the schedule in p, so maps and parameters are built together (conv_prepare) and travel together.
struct ConvLaunch {
  CUtensorMap tmA, tmB;
  ConvParams p;
};

// What an implicit-GEMM launch computes, without its data pointers: conv_select picks its kernel from this alone.
struct ConvRequest {
  yb_conv_desc d;
  // 0 x 0: the forward ksize x ksize window, symmetric padding ksize / 2.  1..2 x 1..2: a kh x kw window whose taps sit
  // at offsets (0..kh-1, 0..kw-1) from the output pixel (zero-filled past the border), stride 1, 16-bit output, output
  // scattered to parity class `scatter` (ConvParams::scatter; the stride-2 dgrad, conv_prepare_dgrad_s2)
  int kh = 0, kw = 0, scatter = 0;
  bool stats = false;      // BN batch statistics of the raw result (stat_sum / stat_sqsum)
  bool res = false;        // adds a residual
  int det_e = 0;           // > 0: detection head with the decode fused into the epilogue, 5 + C = det_e columns per
                           // anchor, d.cout = 3 * det_e <= 256; one n-tile of 64, 128 or 256 columns holds all of them and
                           // `out` is never written
  bool plan_rule = false;  // a forward layer of a 16-bit inference plan: the plan's multicast-cluster rule applies when
                           // YB_CONV_MCAST is unset, and the TMA-store epilogue when YB_CONV_EPI is
};

// The kernel of r, down to its conv_igemm_kernel instantiation, which must exist (no pointers, no device work)
int conv_select(const ConvRequest& r, ConvParams* p);
// conv_select, then the tensor maps over the data pointers.  res and stat_sum / stat_sqsum are given exactly when r asks
// for them; scale = shift = NULL: identity.  Windowed requests take w_packed as [cout_pad][kh*kw*cin].
int conv_prepare(const ConvRequest& r, const void* x, const void* w_packed, const float* scale, const float* shift,
                 const void* res, void* out, float* stat_sum, float* stat_sqsum, ConvLaunch* l);
// Stride-2 dgrad parity class c = 2a + b, the input-gradient pixels (2i + a, 2j + b): its (1 + a) x (1 + b) window's
// [cin_pad][taps * k_cout] weight matrix starts {0, 1, 3, 5}[c] x cin_pad x k_cout elements into the packed weights
// (yb_pack_dgrad_weights_s2), which hold the 9 taps exactly once
inline size_t dgrad_s2_class_offset(int c, int cin_pad, int k_cout) {
  static constexpr int first[4] = {0, 1, 3, 5};
  return (size_t)first[c] * cin_pad * k_cout;
}
// The data gradient of a 3x3 stride-2 conv `fwd` as the four parity-class window convs over the plain dz
// [n, h / 2, w / 2, dz_ld], each scattered into its quarter of dx [n, h, w, dx_ld] (+ res, nullable).  l: [4].
int conv_prepare_dgrad_s2(const yb_conv_desc* fwd, const void* dz, int dz_ld, int k_cout, const void* w_dgrad_s2,
                          const void* res, int res_ld, void* dx, int dx_ld, ConvLaunch* l);
// halo-tile conv for the Cin <= 64 3x3 layers (csrc/conv_halo.cu)
// out: the 16-bit output as {C, W, H, N} = [n, ho, wo, out_ld], one {64, 8, 2, 1} box per consumer warp and 64 channels
// (the TMA-store epilogue; zeroed for an e4m3 output)
struct HaloMaps { CUtensorMap plane[4]; CUtensorMap w; CUtensorMap in3d; CUtensorMap res; CUtensorMap out; };
struct HaloParams {
  int n, ho, wo;               // output geometry
  int tiles_x, tiles_y, num_tiles;
  int cout;
  int leaky;
  const float* scale;
  const float* shift;
  const void* res;             // nullable, [n, ho, wo, res_ld]
  long res_ld;
  void* out;                   // [n, ho, wo, out_ld]
  long out_ld;
  // fused stem (darknet53_body/Conv 3->32 computed on the fly as the producer of Conv_1's halo planes)
  const float* stem_w;         // [32][27] float32 OHWI, NULL: plain halo conv
  const float* stem_scale;     // [32]
  const float* stem_shift;     // [32]
  int in_h, in_w;              // image size (= the stem's output size)
  // 1: the output is e4m3 codes of value * out_inv_scale (Conv_3 of the fp8 plan: fp16 in, e4m3 out)
  int out_e4m3;
  float out_inv_scale;
  int res_smem;                // 1: the residual is TMA-loaded with each tile's halo (Conv_3's shape; YB_CONV_RES)
  // The rest of the conv_halo_kernel instantiation halo_select picks (cout, out_e4m3 and res_smem above are the others);
  // host only, after every field the kernel reads.
  int dtype;                   // yb_dtype of the input and the weights
  int cin, stride;
  int stem;                    // 1: the stem fused in (stem_w ...)
};
// What a halo-tile launch computes, without its data pointers: halo_select picks its kernel from this alone.
struct HaloRequest {
  yb_conv_desc d;
  bool res = false;        // adds a residual
  bool out_e4m3 = false;   // the output is e4m3 codes of value * out_inv_scale (Conv_3 of the fp8 plan: fp16 in)
  bool stem = false;       // the stem (3->32, 3x3/1, BN + leaky) fused into Conv_1 (32->64, 3x3/2): d describes Conv_1,
                           // whose input, the stem's output, is never written; the input is the float32 image [n, d.h, d.w, 3]
};
// One halo-tile launch (host only): the tensor maps and the parameters they were encoded for.
struct HaloLaunch {
  HaloMaps maps;
  HaloParams p;
};
// The kernel of r, down to its conv_halo_kernel instantiation, which must exist (no pointers, no device work)
int halo_select(const HaloRequest& r, HaloParams* p);
// halo_select of the plain request (no residual, 16-bit output, no fused stem) succeeds
bool conv_halo_supported(const yb_conv_desc* d);
// halo_select, then the tensor maps over the data pointers.  x is the input activation, or with r.stem the image;
// res is given exactly when r asks for it, stem_w [32][27] OHWI, stem_scale and stem_shift [32] exactly with r.stem.
int conv_halo_prepare(const HaloRequest& r, const void* x, const void* w_packed, const float* scale, const float* shift,
                      const void* res, void* out, const float* stem_w, const float* stem_scale, const float* stem_shift,
                      HaloLaunch* l);
int conv_halo_launch(const HaloLaunch& l, cudaStream_t st);
// weight gradient of a conv (csrc/conv_wgrad.cu)
struct WgradParams {
  long P;              // output pixels n*ho*wo
  int ho, wo;
  int cin, cout, ksize, stride, pad;
  int kb_per_split;    // 64-pixel blocks per CTA
  int num_kb;          // ceil(P / 64)
  int n_chunks;        // cin / BNW
  int a_dilated;       // dz lives zero-inserted in an [n, 2ho, 2wo, cout] buffer (stride-2 layers): gather it by im2col
  float* dw;           // [cout, k*k*cin] fp32, accumulated
  // The conv_wgrad_kernel instantiation and grid wgrad_select picks; host only, after every field the kernel reads.
  int dtype;           // yb_dtype of x and dz
  int bnw, tp;         // input channels per tap and tile, filter taps per CTA
  int grid_x, grid_y, grid_z;   // pixel splits, tap groups x input-channel chunks, 128-row output-channel tiles
};
struct WgradLaunch {
  CUtensorMap tmA, tmB;
  WgradParams p;
};
// The kernel and grid of the weight gradient of the conv d on a device with sm_count SMs, with the current options
// (YB_WGRAD_TP, YB_WGRAD_EPI, YB_WGRAD_SPLITS; no pointers, no device work)
int wgrad_select(const yb_conv_desc* d, int sm_count, WgradParams* p);
// wgrad_select for the current device, then the tensor maps over x, dz [rows, dz_ld] (dz_dilated: zero-inserted, see
// yb_conv2d_wgrad) and dw
int wgrad_prepare(const yb_conv_desc* d, const void* x, const void* dz, int dz_ld, int dz_dilated, float* dw,
                  WgradLaunch* l);
int wgrad_launch(const WgradLaunch& l, cudaStream_t st);
int conv_launch(const ConvLaunch& l, cudaStream_t st);
// what conv_launch would launch on the current device, without launching: grid (CTAs) and the most clusters of
// p.cluster CTAs that can be resident at once (cudaOccupancyMaxActiveClusters; the SM count when p.cluster == 1)
int conv_launch_grid(const ConvParams& p, int* grid, int* max_clusters);
// the persistent grid for sms SMs of which at most max_clusters clusters are resident (<= 0: sms / cluster)
int conv_grid(const ConvParams& p, int sms, int max_clusters);
// work units: one per cluster of (cluster / cluster_n) m-tiles x cluster_n n-tiles
int conv_units(const ConvParams& p);

}  // namespace yb
