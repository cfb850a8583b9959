// Network plan: Darknet-53 + 3-scale YOLOv3 head (model.py:30-80, utils/layer_utils.py:24-79)
// for a fixed (batch, H, W, dtype): layer schedule, activation/parameter arena layout,
// TMA tensor maps.  concat (model.py:62,72) and NN-upsample (utils/layer_utils.py:82-87)
// never run as ops: producers store straight into channel slices of the concat buffers.
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

#include "common.cuh"
#include "conv.cuh"

#include "net.cuh"

namespace yb {
void train_layout(yb_net* net);
int train_bind(yb_net* net, cudaStream_t st);
int train_refresh_dgrad_weights(yb_net* net, int layer, void* stream);
int nms_candidate_buffers(void* workspace, size_t workspace_bytes, int n_images, int num_boxes, int num_classes,
                          int max_boxes, int** cand_count, float** cand_score, int** cand_idx);
int fp8_fold(const float* gamma, const float* beta, const float* mean, const float* var, int c, float eps, float s_in,
             const float* w_scale, float* scale, float* shift, cudaStream_t st);
int nms_select_gather(const float* boxes, int n_images, int num_boxes, int num_classes, int max_boxes, float iou_thresh,
                      void* workspace, size_t workspace_bytes, float* out_boxes, float* out_scores, int32_t* out_labels,
                      int32_t* out_indices, int32_t* out_counts, cudaStream_t st);

static size_t align256(size_t v) { return (v + 255) & ~size_t(255); }

// fp8 plan: the stem, Conv_1, Conv_2 and Conv_3 (layers 0-3) stay fp16 (HBM-bound kernels with no e4m3 variant, ~5 %
// of the FLOPs); Conv_3 writes the first e4m3 buffer, every later conv reads and writes e4m3 (heads: fp32 out).
static constexpr int FP8_FIRST_LAYER = 4;
static bool layer_is_e4m3(const yb_net* net, int i) { return net->dtype == YB_E4M3 && i >= FP8_FIRST_LAYER; }

struct Builder {
  yb_net* net;
  int body_k = 0, head_k = 0;

  int new_buf(int h, int w, int ld, int fp32) {
    Buf b; b.h = h; b.w = w; b.ld = ld; b.fp32 = fp32;
    net->bufs.push_back(b);
    return (int)net->bufs.size() - 1;
  }
  // conv2d of utils/layer_utils.py:9-22.  dst: optional pre-allocated destination view.
  Ten conv(const Ten& x, int cout, int k, int s, bool head, bool bn = true, const Ten* shortcut = nullptr,
           const Ten* dst = nullptr, bool upsample = false) {
    Layer L;
    memset(&L.info, 0, sizeof(L.info));
    L.info.index = (int)net->layers.size();
    L.info.cin = x.c; L.info.cout = cout; L.info.ksize = k; L.info.stride = s; L.info.has_bn = bn ? 1 : 0;
    L.info.in_h = x.h; L.info.in_w = x.w; L.info.out_h = x.h / s; L.info.out_w = x.w / s;
    L.info.is_head = head ? 1 : 0;
    L.info.scope_index = head ? head_k++ : body_k++;
    L.in = x;
    L.upsample = upsample;
    L.info.upsample2x = upsample ? 1 : 0;
    L.out_fp32 = !bn;
    L.cout_pad = yb_conv_cout_pad(cout);
    if (shortcut) L.res = *shortcut; else L.res.buf = -2;
    Ten y;
    if (dst) {
      y = *dst;
    } else {
      y.buf = new_buf(x.h / s, x.w / s, cout, !bn);
      y.off = 0;
    }
    y.c = cout;
    y.h = (x.h / s) * (upsample ? 2 : 1);
    y.w = (x.w / s) * (upsample ? 2 : 1);
    L.out = y;
    net->layers.push_back(L);
    return y;
  }
  Ten res_block(const Ten& x, int f, const Ten* dst = nullptr) {   // utils/layer_utils.py:25-32
    Ten a = conv(x, f, 1, 1, false);
    return conv(a, 2 * f, 3, 1, false, true, &x, dst);
  }
  void yolo_block(const Ten& x, int f, Ten* route, Ten* net_out) {  // utils/layer_utils.py:71-79
    Ten t = conv(x, f, 1, 1, true);
    t = conv(t, 2 * f, 3, 1, true);
    t = conv(t, f, 1, 1, true);
    t = conv(t, 2 * f, 3, 1, true);
    t = conv(t, f, 1, 1, true);
    *route = t;
    *net_out = conv(t, 2 * f, 3, 1, true);
  }

  void build() {
    const int H = net->h, W = net->w, D = 3 * (5 + net->class_num);
    // concat buffers (model.py:62,72): [upsampled | route]
    const int cat1 = new_buf(H / 16, W / 16, 256 + 512, 0);
    const int cat2 = new_buf(H / 8, W / 8, 128 + 256, 0);
    Ten x; x.buf = -1; x.c = 3; x.h = H; x.w = W;
    // ---- darknet53_body (utils/layer_utils.py:35-66) ----
    Ten t = conv(x, 32, 3, 1, false);
    t = conv(t, 64, 3, 2, false);
    t = res_block(t, 32);
    t = conv(t, 128, 3, 2, false);
    for (int i = 0; i < 2; ++i) t = res_block(t, 64);
    t = conv(t, 256, 3, 2, false);
    Ten r1dst; r1dst.buf = cat2; r1dst.off = 128;
    for (int i = 0; i < 8; ++i) t = res_block(t, 128, i == 7 ? &r1dst : nullptr);
    const Ten route1 = t;
    t = conv(t, 512, 3, 2, false);
    Ten r2dst; r2dst.buf = cat1; r2dst.off = 256;
    for (int i = 0; i < 8; ++i) t = res_block(t, 256, i == 7 ? &r2dst : nullptr);
    const Ten route2 = t;
    t = conv(t, 1024, 3, 2, false);
    for (int i = 0; i < 4; ++i) t = res_block(t, 512);
    const Ten route3 = t;
    (void)route1; (void)route2;
    // ---- yolov3_head (model.py:53-78) ----
    Ten inter, nt;
    yolo_block(route3, 512, &inter, &nt);
    Ten fm1 = conv(nt, D, 1, 1, true, false);
    Ten up1; up1.buf = cat1; up1.off = 0;
    conv(inter, 256, 1, 1, true, true, nullptr, &up1, true);
    Ten c1; c1.buf = cat1; c1.off = 0; c1.c = 768; c1.h = H / 16; c1.w = W / 16;
    yolo_block(c1, 256, &inter, &nt);
    Ten fm2 = conv(nt, D, 1, 1, true, false);
    Ten up2; up2.buf = cat2; up2.off = 0;
    conv(inter, 128, 1, 1, true, true, nullptr, &up2, true);
    Ten c2; c2.buf = cat2; c2.off = 0; c2.c = 384; c2.h = H / 8; c2.w = W / 8;
    yolo_block(c2, 128, &inter, &nt);
    Ten fm3 = conv(nt, D, 1, 1, true, false);
    net->fm_buf[0] = fm1.buf; net->fm_buf[1] = fm2.buf; net->fm_buf[2] = fm3.buf;

    // ---- arenas ----
    const bool fp8 = net->dtype == YB_E4M3;
    for (auto& b : net->bufs) b.esz = b.fp32 ? 4 : (fp8 ? 1 : 2);
    for (int i = 0; fp8 && i < FP8_FIRST_LAYER - 1; ++i) net->bufs[net->layers[i].out.buf].esz = 2;
    net->buf_scale.assign(net->bufs.size(), 1.f);
    size_t o = 0;
    for (auto& b : net->bufs) {
      b.bytes = (size_t)net->n * b.h * b.w * b.ld * b.esz;
      b.offset = o;
      o = align256(o + b.bytes);
    }
    net->act_bytes = o;
    o = 0;
    for (auto& L : net->layers) {
      const bool q = layer_is_e4m3(net, L.info.index);
      L.dtype = q ? YB_E4M3 : (fp8 ? YB_F16 : net->dtype);
      const size_t kk = (size_t)L.info.ksize * L.info.ksize * L.info.cin;
      L.w_master = o; o = align256(o + (size_t)L.info.cout * kk * 4);
      L.w_packed = o; o = align256(o + (size_t)L.cout_pad * kk * (q ? 1 : 2));
      if (q) { L.w_scale = o; o = align256(o + (size_t)L.cout_pad * 4); }
      const size_t cb = (size_t)L.cout_pad * 4;
      if (L.info.has_bn) {
        L.gamma = o; o = align256(o + cb);
        L.beta = o;  o = align256(o + cb);
        L.mean = o;  o = align256(o + cb);
        L.var = o;   o = align256(o + cb);
      } else {
        L.bias = o;  o = align256(o + cb);
      }
      L.scale = o; o = align256(o + cb);
      if (L.info.has_bn) { L.shift = o; o = align256(o + cb); }
      else L.shift = L.bias;   // detection convs: the epilogue's shift IS the (trainable) bias
    }
    net->param_bytes = o;
  }
};

void* ten_ptr(const yb_net* net, const Ten& t) {
  const Buf& b = net->bufs[t.buf];
  return net->act + b.offset + (size_t)t.off * b.esz;
}

// e4m3 plan: each layer's residual and output scales come from its buffers (host-side launch parameters)
static void apply_fp8_scales(yb_net* net) {
  for (size_t i = FP8_FIRST_LAYER - 1; i < net->layers.size(); ++i) {
    Layer& L = net->layers[i];
    const float so = net->buf_scale[L.out.buf];
    L.fwd.p.res_scale = L.res.buf >= 0 ? net->buf_scale[L.res.buf] : 1.f;
    L.fwd.p.out_inv_scale = 1.f / so;
    L.halo.p.out_inv_scale = 1.f / so;
  }
}

// e4m3 layer: scale = (BN scale) x s_in x s_w[c] (the detection heads' shift is their bias)
static int fold_e4m3_layer(yb_net* net, Layer& L, cudaStream_t st) {
  const bool bn = L.info.has_bn;
  auto f = [&](size_t off) { return reinterpret_cast<float*>(net->par + off); };
  return fp8_fold(bn ? f(L.gamma) : nullptr, bn ? f(L.beta) : nullptr, bn ? f(L.mean) : nullptr, bn ? f(L.var) : nullptr,
                  L.info.cout, net->bn_eps, net->buf_scale[L.in.buf], f(L.w_scale), f(L.scale), f(L.shift), st);
}

yb_conv_desc layer_desc(const yb_net* net, const Layer& L) {
  yb_conv_desc d;
  memset(&d, 0, sizeof(d));
  d.n = net->n; d.h = L.info.in_h; d.w = L.info.in_w; d.cin = L.info.cin; d.cout = L.info.cout;
  d.ksize = L.info.ksize; d.stride = L.info.stride;
  d.in_ld = net->bufs[L.in.buf].ld; d.out_ld = net->bufs[L.out.buf].ld;
  d.res_ld = L.res.buf >= 0 ? net->bufs[L.res.buf].ld : 0;
  d.dtype = L.dtype; d.out_fp32 = L.out_fp32; d.leaky = L.info.has_bn; d.upsample2x = L.upsample;
  return d;
}
// the multicast-cluster rule of conv_select applies to the 16-bit inference plans (not training, not e4m3)
static bool plan_mcast_rule(const yb_net* net) { return !net->training && net->dtype != YB_E4M3; }
// The halo-tile request of layer i's inference forward: Conv_3 of the fp8 plan reads fp16 and writes e4m3
static HaloRequest layer_halo_request(const yb_net* net, int i) {
  const Layer& L = net->layers[i];
  HaloRequest r{layer_desc(net, L)};
  r.res = L.res.buf >= 0;
  r.out_e4m3 = net->dtype == YB_E4M3 && i == FP8_FIRST_LAYER - 1;
  return r;
}

// What the forward launches for layer i.  It reads the options at every call: they may change between forwards of
// one bound plan.  Layer 0 is FusedStem when layer 1's launch computes it; it then has no launch of its own.
enum class LayerKernel { FusedStem, Stem, Thin, Halo, Igemm };
static LayerKernel layer_kernel(const yb_net* net, int i) {
  if (i == 0) return layer_kernel(net, 1) == LayerKernel::FusedStem ? LayerKernel::FusedStem : LayerKernel::Stem;
  const Layer& L = net->layers[i];
  // Cin = 32: 64-byte im2col rows halve the TMA line rate -> the mma.sync halo-tile kernel (csrc/conv_thin.cu), opt-in
  // (YB_THIN=2); by default these layers take the tensor-core path
  if (opt("YB_THIN")[0] == '2' && net->dtype != YB_E4M3 && L.info.ksize == 3 && L.info.cin == 32 && L.info.has_bn &&
      !L.upsample)
    return LayerKernel::Thin;
  const yb_conv_desc d = layer_desc(net, L);
  if (!conv_halo_supported(&d)) return LayerKernel::Igemm;
  // halo-tile kernel: default on for Cin = 32, whose 64-byte im2col rows make the implicit GEMM TMA-row bound; the
  // 64->128 layers leave room for only two halo stages beside their weights.  YB_HALO=0: never, YB_HALO=1: wherever
  // supported.  The fp8 plan's Conv_3 always runs it: only it writes e4m3 from fp16.
  const char* hopt = opt("YB_HALO");
  // stem fused into Conv_1 (csrc/conv_halo.cu): layer 0's output is never written.  YB_STEM_FUSE=0: two launches.
  if (i == 1 && L.info.cin == 32 && L.info.stride == 2 && hopt[0] != '0' && opt("YB_STEM_FUSE")[0] != '0')
    return LayerKernel::FusedStem;
  if ((net->dtype == YB_E4M3 && i == FP8_FIRST_LAYER - 1) || (hopt[0] != '0' && (hopt[0] == '1' || L.info.cin == 32)))
    return LayerKernel::Halo;
  return LayerKernel::Igemm;
}

__global__ void fill_kernel(float* p, int n, float v) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}

}  // namespace yb

using namespace yb;

extern "C" int yb_net_create(yb_net** out, int class_num, int n, int h, int w, int dtype, int training) {
  YB_REQUIRE(out, "net_create: null out pointer");
  YB_REQUIRE(class_num > 0 && n > 0, "net_create: bad class_num/batch");
  YB_REQUIRE(h > 0 && w > 0 && h % 32 == 0 && w % 32 == 0, "net_create: H,W must be multiples of 32 (got %dx%d)", h, w);
  YB_REQUIRE(dtype == YB_F16 || dtype == YB_BF16 || dtype == YB_E4M3, "net_create: dtype must be f16, bf16 or e4m3");
  YB_REQUIRE(!(dtype == YB_E4M3 && training), "net_create: e4m3 is an inference plan (quantize a trained fp16/bf16 model)");
  yb_net* net = new yb_net();
  net->class_num = class_num; net->n = n; net->h = h; net->w = w; net->dtype = dtype; net->training = training;
  Builder b{net};
  b.build();
  if (training) train_layout(net);
  *out = net;
  return YB_OK;
}

extern "C" int yb_net_destroy(yb_net* net) { delete net; return YB_OK; }

extern "C" int yb_net_num_layers(const yb_net* net) { return net ? (int)net->layers.size() : YB_ERR_INVALID_ARGUMENT; }

extern "C" int yb_net_layer_info(const yb_net* net, int layer, yb_layer_info* info) {
  YB_REQUIRE(net && info && layer >= 0 && layer < (int)net->layers.size(), "layer_info: bad argument");
  *info = net->layers[layer].info;
  return YB_OK;
}

extern "C" int yb_net_layer_schedule(const yb_net* net, int layer, int sm_count, yb_layer_schedule_info* info) {
  YB_REQUIRE(net && info && layer >= 0 && layer < (int)net->layers.size() && sm_count >= 0, "layer_schedule: bad argument");
  memset(info, 0, sizeof(*info));
  const LayerKernel k = layer_kernel(net, layer);
  switch (k) {
    case LayerKernel::FusedStem: info->kernel = YB_LAYER_FUSED_STEM; break;
    case LayerKernel::Stem: info->kernel = YB_LAYER_STEM; break;
    case LayerKernel::Thin: info->kernel = YB_LAYER_THIN; break;
    case LayerKernel::Halo: info->kernel = YB_LAYER_HALO; break;
    case LayerKernel::Igemm: info->kernel = YB_LAYER_IGEMM; break;
  }
  if (layer == 0) return YB_OK;                        // the stem
  const Layer& L = net->layers[layer];
  const yb_conv_desc d = layer_desc(net, L);
  info->residual = L.res.buf >= 0 ? 1 : 0;
  if (k == LayerKernel::Halo) {
    HaloParams hp;
    int rc = halo_select(layer_halo_request(net, layer), &hp);
    if (rc) return rc;
    info->res_smem = hp.res_smem;
  }
  if (k != LayerKernel::Igemm) return YB_OK;           // the thin, halo and fused-stem kernels
  ConvRequest r{d};
  r.res = info->residual;
  r.plan_rule = plan_mcast_rule(net);
  ConvParams p;
  int rc = conv_select(r, &p);
  if (rc) return rc;
  if (!L.info.has_bn && 3 * (5 + net->class_num) <= 256) {   // the head's fused-decode launch (yb_net_detect)
    ConvRequest rd{d};
    rd.det_e = 5 + net->class_num;
    ConvParams pd;
    rc = conv_select(rd, &pd);
    if (rc) return rc;
    info->det_block_n = pd.block_n;
  }
  info->igemm = 1;
  info->res_smem = p.res_smem;
  info->epi_tma = p.epi_tma;
  info->pingpong = p.pingpong;
  info->cluster_m = p.cluster / p.cluster_n;
  info->cluster_n = p.cluster_n;
  info->block_m = 64 * p.consumers;
  info->block_n = p.block_n;
  info->num_m_tiles = p.num_m_tiles;
  info->num_n_tiles = p.num_n_tiles;
  info->units = conv_units(p);
  if (sm_count > 0) {
    info->max_clusters = sm_count / p.cluster;
    info->grid = conv_grid(p, sm_count, 0);
    return YB_OK;
  }
  return conv_launch_grid(p, &info->grid, &info->max_clusters);
}

extern "C" int yb_net_arena_bytes(const yb_net* net, size_t* activation_bytes, size_t* param_bytes) {
  YB_REQUIRE(net && activation_bytes && param_bytes, "arena_bytes: bad argument");
  *activation_bytes = net->act_bytes;
  *param_bytes = net->param_bytes;
  return YB_OK;
}

extern "C" int yb_net_bind(yb_net* net, void* activation_arena, size_t activation_bytes, void* param_arena,
                           size_t param_bytes, void* stream) {
  YB_REQUIRE(net && activation_arena && param_arena, "bind: null pointer");
  YB_REQUIRE(activation_bytes >= net->act_bytes && param_bytes >= net->param_bytes, "bind: arena too small");
  YB_REQUIRE(((uintptr_t)activation_arena & 255) == 0 && ((uintptr_t)param_arena & 255) == 0,
             "bind: arenas must be 256-byte aligned");
  net->act = static_cast<uint8_t*>(activation_arena);
  net->par = static_cast<uint8_t*>(param_arena);
  // prepare every tensor-core conv (layer 0 is the CUDA-core stem)
  for (size_t i = 1; i < net->layers.size(); ++i) {
    Layer& L = net->layers[i];
    yb_conv_desc d = layer_desc(net, L);
    const void* res = L.res.buf >= 0 ? ten_ptr(net, L.res) : nullptr;
    const float* scale = reinterpret_cast<const float*>(net->par + L.scale);
    const float* shift = reinterpret_cast<const float*>(net->par + L.shift);
    // every layer layer_kernel may give the halo kernel; Conv_3 of the fp8 plan (fp16 in, e4m3 out) runs nothing else
    const HaloRequest hr = layer_halo_request(net, (int)i);
    if (hr.out_e4m3 || conv_halo_supported(&d)) {
      int rc = conv_halo_prepare(hr, ten_ptr(net, L.in), net->par + L.w_packed, scale, shift, res, ten_ptr(net, L.out),
                                 nullptr, nullptr, nullptr, &L.halo);
      if (rc) return rc;
      if (hr.out_e4m3) continue;
    }
    ConvRequest r{d};
    r.res = res != nullptr;
    r.plan_rule = plan_mcast_rule(net);
    int rc = conv_prepare(r, ten_ptr(net, L.in), net->par + L.w_packed, scale, shift, res, ten_ptr(net, L.out), nullptr,
                          nullptr, &L.fwd);
    if (rc) return rc;
    if (!L.info.has_bn) {
      // fused-decode variant of the head (yb_net_detect), for 1 to 80 classes; more keep the unfused pipeline
      ConvRequest rd{d};
      rd.det_e = 5 + net->class_num;
      void* x = ten_ptr(net, L.in);
      L.det_ok = conv_prepare(rd, x, net->par + L.w_packed, scale, shift, nullptr, x /* never written */, nullptr, nullptr,
                              &L.det) == YB_OK;
    }
  }
  if (net->fp8_ready) apply_fp8_scales(net);
  if (net->training) return train_bind(net, static_cast<cudaStream_t>(stream));
  return YB_OK;
}

extern "C" int yb_net_set_conv_params(yb_net* net, int layer, const float* w, int layout, const float* gamma,
                                      const float* beta, const float* mean, const float* var, const float* bias,
                                      void* stream) {
  YB_REQUIRE(net && net->par, "set_conv_params: net not bound");
  YB_REQUIRE(layer >= 0 && layer < (int)net->layers.size() && w, "set_conv_params: bad argument");
  Layer& L = net->layers[layer];
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int c = L.info.cout;
  int rc = yb_pack_conv_weights(w, layout, c, L.info.cin, L.info.ksize, c, YB_F32, net->par + L.w_master, stream);
  if (rc) return rc;
  const bool q = L.dtype == YB_E4M3;
  rc = q ? yb_pack_conv_weights_e4m3(w, layout, c, L.info.cin, L.info.ksize, L.cout_pad, net->par + L.w_packed,
                                     reinterpret_cast<float*>(net->par + L.w_scale), stream)
         : yb_pack_conv_weights(w, layout, c, L.info.cin, L.info.ksize, L.cout_pad, L.dtype, net->par + L.w_packed, stream);
  if (rc) return rc;
  float* scale = reinterpret_cast<float*>(net->par + L.scale);
  float* shift = reinterpret_cast<float*>(net->par + L.shift);
  if (L.info.has_bn) {
    YB_REQUIRE(gamma && beta && mean && var, "set_conv_params: layer %d needs gamma/beta/mean/var", layer);
    YB_CUDA(cudaMemcpyAsync(net->par + L.gamma, gamma, c * 4, cudaMemcpyDeviceToDevice, st));
    YB_CUDA(cudaMemcpyAsync(net->par + L.beta, beta, c * 4, cudaMemcpyDeviceToDevice, st));
    YB_CUDA(cudaMemcpyAsync(net->par + L.mean, mean, c * 4, cudaMemcpyDeviceToDevice, st));
    YB_CUDA(cudaMemcpyAsync(net->par + L.var, var, c * 4, cudaMemcpyDeviceToDevice, st));
    rc = yb_bn_fold(gamma, beta, mean, var, c, 1e-5f, scale, shift, stream);   // model.py:37 epsilon
    if (rc) return rc;
  } else {
    YB_REQUIRE(bias, "set_conv_params: layer %d needs a bias", layer);
    YB_CUDA(cudaMemsetAsync(shift, 0, L.cout_pad * 4, st));          // shift aliases the bias buffer
    YB_CUDA(cudaMemcpyAsync(net->par + L.bias, bias, c * 4, cudaMemcpyDeviceToDevice, st));
    fill_kernel<<<ceil_div(L.cout_pad, 128), 128, 0, st>>>(scale, L.cout_pad, 1.0f);
    YB_CUDA(cudaGetLastError());
  }
  if (q) {
    rc = fold_e4m3_layer(net, L, st);
    if (rc) return rc;
  }
  if (net->training) return train_refresh_dgrad_weights(net, layer, stream);
  return YB_OK;
}

extern "C" int yb_net_refold_bn(yb_net* net, void* stream) {
  YB_REQUIRE(net && net->par, "refold_bn: net not bound");
  for (auto& L : net->layers) {
    if (L.dtype == YB_E4M3) {
      int rc = fold_e4m3_layer(net, L, static_cast<cudaStream_t>(stream));
      if (rc) return rc;
      continue;
    }
    if (!L.info.has_bn) continue;
    int rc = yb_bn_fold(reinterpret_cast<const float*>(net->par + L.gamma), reinterpret_cast<const float*>(net->par + L.beta),
                        reinterpret_cast<const float*>(net->par + L.mean), reinterpret_cast<const float*>(net->par + L.var),
                        L.info.cout, net->bn_eps, reinterpret_cast<float*>(net->par + L.scale),
                        reinterpret_cast<float*>(net->par + L.shift), stream);
    if (rc) return rc;
  }
  net->fold_dirty = false;
  return YB_OK;
}

extern "C" int yb_net_forward(yb_net* net, const float* images, float* fm1, float* fm2, float* fm3, void* stream) {
  return yb_net_forward_layers(net, images, fm1, fm2, fm3, 0, 1 << 30, stream);
}

static int forward_layers_impl(yb_net* net, const float* images, float* fm1, float* fm2, float* fm3, int first, int last,
                               const DetParams* det /* [3] or NULL */, void* stream);

extern "C" int yb_net_forward_layers(yb_net* net, const float* images, float* fm1, float* fm2, float* fm3, int first,
                                     int last, void* stream) {
  return forward_layers_impl(net, images, fm1, fm2, fm3, first, last, nullptr, stream);
}

static int forward_layers_impl(yb_net* net, const float* images, float* fm1, float* fm2, float* fm3, int first, int last,
                               const DetParams* det, void* stream) {
  YB_REQUIRE(net && net->act && net->par, "forward: net not bound");
  YB_REQUIRE(images, "forward: null images");
  YB_REQUIRE(first >= 0 && first <= last, "forward: bad layer range");
  YB_REQUIRE(net->dtype != YB_E4M3 || net->fp8_ready,
             "forward: the e4m3 plan has no activation scales (yb_net_set_fp8_amax after calibration)");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  float* user_fm[3] = {fm1, fm2, fm3};
  if (net->fold_dirty) {   // BN parameters / moving statistics changed by a training step: refold for inference
    int rc = yb_net_refold_bn(net, stream);
    if (rc) return rc;
  }
  const bool thin = opt("YB_THIN")[0] != '0';   // A/B switch for the thin-layer kernels
  // detect path: heads 1 and 2 on a side stream (YB_HEAD_STREAM=0: everything on the caller's stream)
  const bool head_overlap = det != nullptr && opt("YB_HEAD_STREAM")[0] != '0';
  bool forked = false;
  if (head_overlap && net->side_stream == nullptr) {
    YB_CUDA(cudaStreamCreateWithFlags(&net->side_stream, cudaStreamNonBlocking));
    YB_CUDA(cudaEventCreateWithFlags(&net->side_fork, cudaEventDisableTiming));
    YB_CUDA(cudaEventCreateWithFlags(&net->side_join, cudaEventDisableTiming));
  }
  for (size_t i = first; i < net->layers.size() && (int)i <= last; ++i) {
    Layer& L = net->layers[i];
    const LayerKernel k = layer_kernel(net, (int)i);
    if (k != LayerKernel::Igemm) {   // (layer 0 under FusedStem: nothing, layer 1's launch computes it)
      int rc = YB_OK;
      if (k == LayerKernel::Stem && thin) {
        rc = yb_stem_conv_fwd_tc(images, reinterpret_cast<const float*>(net->par + L.w_master),
                                 reinterpret_cast<const float*>(net->par + L.scale),
                                 reinterpret_cast<const float*>(net->par + L.shift), net->n, net->h, net->w, L.dtype, 1,
                                 ten_ptr(net, L.out), stream);
      } else if (k == LayerKernel::Stem) {
        rc = yb_stem_conv_fwd(images, reinterpret_cast<const float*>(net->par + L.w_master),
                              reinterpret_cast<const float*>(net->par + L.scale),
                              reinterpret_cast<const float*>(net->par + L.shift), net->n, net->h, net->w, L.info.cout,
                              L.dtype, 1, ten_ptr(net, L.out), stream);
      } else if (k == LayerKernel::Thin) {
        const yb_conv_desc d = layer_desc(net, L);
        rc = yb_conv3x3_thin_fwd(&d, ten_ptr(net, L.in), net->par + L.w_packed,
                                 reinterpret_cast<const float*>(net->par + L.scale),
                                 reinterpret_cast<const float*>(net->par + L.shift),
                                 L.res.buf >= 0 ? ten_ptr(net, L.res) : nullptr, ten_ptr(net, L.out), stream);
      } else if (k == LayerKernel::FusedStem && i == 1) {
        // per forward: the image is an argument of the forward
        Layer& L0 = net->layers[0];
        HaloRequest r{layer_desc(net, L)};
        r.stem = true;
        HaloLaunch hl;
        rc = conv_halo_prepare(r, images, net->par + L.w_packed, reinterpret_cast<const float*>(net->par + L.scale),
                               reinterpret_cast<const float*>(net->par + L.shift), nullptr, ten_ptr(net, L.out),
                               reinterpret_cast<const float*>(net->par + L0.w_master),
                               reinterpret_cast<const float*>(net->par + L0.scale),
                               reinterpret_cast<const float*>(net->par + L0.shift), &hl);
        if (rc == YB_OK) rc = conv_halo_launch(hl, st);
      } else if (k == LayerKernel::Halo) {
        rc = conv_halo_launch(L.halo, st);
      }
      if (rc) return rc;
      continue;
    }
    if (!L.info.has_bn) {
      int which = L.out.buf == net->fm_buf[0] ? 0 : (L.out.buf == net->fm_buf[1] ? 1 : 2);
      if (det) {                                      // decode + candidate filter in the epilogue, no feature map
        ConvLaunch dl = L.det;
        dl.p.det = det[which];
        // The first two heads are leaves of the graph (nothing but the NMS reads what they produce) and small (43 / 170
        // tiles): they run on the plan's side stream beside the upsampling branch that continues on the caller's stream;
        // the last head is on the critical path.  Every layer output has its own buffer, so the head's input stays intact.
        cudaStream_t hs = st;
        if (head_overlap && which < 2) {
          YB_CUDA(cudaEventRecord(net->side_fork, st));
          YB_CUDA(cudaStreamWaitEvent(net->side_stream, net->side_fork, 0));
          hs = net->side_stream;
          forked = true;
        }
        int rc = conv_launch(dl, hs);
        if (rc) return rc;
        continue;
      }
      L.fwd.p.out = user_fm[which] ? (void*)user_fm[which] : ten_ptr(net, L.out);
    }
    int rc = conv_launch(L.fwd, st);
    if (rc) return rc;
  }
  if (forked) {
    YB_CUDA(cudaEventRecord(net->side_join, net->side_stream));
    YB_CUDA(cudaStreamWaitEvent(st, net->side_join, 0));
  }
  return YB_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// forward -> predict -> score = conf * prob -> per-image gpu_nms in one call (test_single_image.py:50-57): the decode and
// the score filter run inside the three detection-head epilogues, then the greedy selection reads the candidate lists.
// ---------------------------------------------------------------------------------------------------------------
static int det_num_boxes(const yb_net* net) {
  int b = 0;
  for (int s = 0; s < 3; ++s) b += 3 * (net->h / (32 >> s)) * (net->w / (32 >> s));
  return b;
}

extern "C" int yb_net_detect_supported(const yb_net* net) {
  if (!net || !net->act) return 0;
  for (auto& L : net->layers) if (!L.info.has_bn && !L.det_ok) return 0;
  return 1;
}

extern "C" int yb_net_detect_workspace_bytes(const yb_net* net, int max_boxes, size_t* bytes) {
  YB_REQUIRE(net && bytes && max_boxes >= 0, "detect_workspace_bytes: bad argument");
  return yb_nms_workspace_bytes(net->n, det_num_boxes(net), net->class_num, max_boxes, bytes);
}

extern "C" int yb_net_detect(yb_net* net, const float* images, const float* anchors9x2, int max_boxes, float score_thresh,
                             float iou_thresh, void* workspace, size_t workspace_bytes, float* boxes, float* out_boxes,
                             float* out_scores, int32_t* out_labels, int32_t* out_indices, int32_t* out_counts,
                             void* stream) {
  return yb_net_detect_phases(net, images, anchors9x2, max_boxes, score_thresh, iou_thresh, workspace, workspace_bytes,
                              boxes, out_boxes, out_scores, out_labels, out_indices, out_counts, 7, stream);
}

extern "C" int yb_net_detect_phases(yb_net* net, const float* images, const float* anchors9x2, int max_boxes,
                                    float score_thresh, float iou_thresh, void* workspace, size_t workspace_bytes,
                                    float* boxes, float* out_boxes, float* out_scores, int32_t* out_labels,
                                    int32_t* out_indices, int32_t* out_counts, int phases, void* stream) {
  YB_REQUIRE(net && net->act && net->par, "detect: net not bound");
  YB_REQUIRE(images && anchors9x2 && workspace && boxes && out_counts, "detect: null pointer");
  YB_REQUIRE(max_boxes >= 0, "detect: bad max_boxes");
  if (!yb_net_detect_supported(net)) {
    set_error("detect: no fused-decode kernel for %d classes (use forward + predict + nms)", net->class_num);
    return YB_ERR_UNSUPPORTED;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int n = net->n, B = det_num_boxes(net), C = net->class_num;
  if (max_boxes == 0) {
    YB_CUDA(cudaMemsetAsync(out_counts, 0, sizeof(int32_t) * n, st));
    return YB_OK;
  }
  YB_REQUIRE(out_boxes && out_scores && out_labels && out_indices, "detect: null pointer");
  YB_REQUIRE(((uintptr_t)boxes & 15) == 0 && ((uintptr_t)out_boxes & 15) == 0, "detect: boxes must be 16-byte aligned");
  int* cand_count; float* cand_score; int* cand_idx;
  int rc = nms_candidate_buffers(workspace, workspace_bytes, n, B, C, max_boxes, &cand_count, &cand_score, &cand_idx);
  if (rc) return rc;
  if (phases & 1) YB_CUDA(cudaMemsetAsync(cand_count, 0, sizeof(int) * (size_t)n * C, st));
  DetParams det[3];
  int off = 0;
  for (int s = 0; s < 3; ++s) {
    DetParams& d = det[s];
    memset(&d, 0, sizeof(d));
    const int gh = net->h / (32 >> s), gw = net->w / (32 >> s);
    d.boxes = boxes; d.cand_count = cand_count; d.cand_score = cand_score; d.cand_idx = cand_idx;
    d.B = B; d.C = C; d.E = 5 + C; d.box_off = off;
    off += 3 * gh * gw;
    d.ratio_h = (float)((double)net->h / (double)gh);        // model.py:91 (float64 divide, cast to f32)
    d.ratio_w = (float)((double)net->w / (double)gw);
    for (int a = 0; a < 3; ++a) {                            // anchor groups 6:9, 3:6, 0:3 (model.py:148-150)
      d.anchor_w[a] = anchors9x2[2 * ((2 - s) * 3 + a)];
      d.anchor_h[a] = anchors9x2[2 * ((2 - s) * 3 + a) + 1];
    }
    d.thr = score_thresh;
    // logits below logit(thr) - 0.01 give sigmoid < thr by > 1e-3 (float error ~1e-7): exact pre-filter
    d.logit_lo = (score_thresh > 0.f && score_thresh < 1.f)
                     ? (float)(log((double)score_thresh / (1.0 - (double)score_thresh)) - 0.01) : -INFINITY;
    d.on = 1;
  }
  if (phases & 1) {
    rc = forward_layers_impl(net, images, nullptr, nullptr, nullptr, 0, 0, det, stream);
    if (rc) return rc;
  }
  if (phases & 2) {
    rc = forward_layers_impl(net, images, nullptr, nullptr, nullptr, 1, 1 << 30, det, stream);
    if (rc) return rc;
  }
  if (!(phases & 4)) return YB_OK;
  return nms_select_gather(boxes, n, B, C, max_boxes, iou_thresh, workspace, workspace_bytes, out_boxes, out_scores,
                           out_labels, out_indices, out_counts, st);
}

extern "C" int yb_net_layer_output(const yb_net* net, int layer, void** ptr, int* ld, int* dtype) {
  YB_REQUIRE(net && net->act && layer >= 0 && layer < (int)net->layers.size() && ptr && ld && dtype,
             "layer_output: bad argument");
  const Layer& L = net->layers[layer];
  *ptr = ten_ptr(net, L.out);
  const Buf& b = net->bufs[L.out.buf];
  *ld = b.ld;
  *dtype = b.fp32 ? YB_F32 : (b.esz == 1 ? YB_E4M3 : (net->dtype == YB_E4M3 ? YB_F16 : net->dtype));
  return YB_OK;
}

extern "C" int yb_net_set_fp8_amax(yb_net* net, const float* amax, int count, void* stream) {
  YB_REQUIRE(net && net->par && amax, "set_fp8_amax: net not bound");
  YB_REQUIRE(net->dtype == YB_E4M3, "set_fp8_amax: not an e4m3 plan");
  YB_REQUIRE(count == (int)net->layers.size(), "set_fp8_amax: need one amax per layer (%d, got %d)", (int)net->layers.size(),
             count);
  // a buffer's scale covers every layer that writes it (the concat buffers: the upsampling conv and the route conv)
  std::vector<float> bmax(net->bufs.size(), 0.f);
  for (size_t i = 0; i < net->layers.size(); ++i) {
    YB_REQUIRE(amax[i] >= 0.f && isfinite(amax[i]), "set_fp8_amax: layer %d amax %g is not finite and >= 0", (int)i, amax[i]);
    float& m = bmax[net->layers[i].out.buf];
    m = fmaxf(m, amax[i]);
  }
  for (size_t b = 0; b < net->bufs.size(); ++b)
    net->buf_scale[b] = (net->bufs[b].esz == 1 && bmax[b] > 0.f) ? bmax[b] / 448.f : 1.f;
  net->fp8_ready = true;
  apply_fp8_scales(net);
  return yb_net_refold_bn(net, stream);
}

extern "C" int yb_net_fp8_layer_scales(const yb_net* net, int layer, float* in_res_out, float** w_scale) {
  YB_REQUIRE(net && net->par && layer >= 0 && layer < (int)net->layers.size() && in_res_out && w_scale,
             "fp8_layer_scales: bad argument");
  YB_REQUIRE(net->dtype == YB_E4M3, "fp8_layer_scales: not an e4m3 plan");
  const Layer& L = net->layers[layer];
  in_res_out[0] = L.in.buf >= 0 ? net->buf_scale[L.in.buf] : 1.f;
  in_res_out[1] = L.res.buf >= 0 ? net->buf_scale[L.res.buf] : 1.f;
  in_res_out[2] = net->buf_scale[L.out.buf];
  *w_scale = L.dtype == YB_E4M3 ? reinterpret_cast<float*>(net->par + L.w_scale) : nullptr;
  return YB_OK;
}

extern "C" int yb_net_forward_launches(const yb_net* net) { return net ? (int)net->layers.size() : 0; }
