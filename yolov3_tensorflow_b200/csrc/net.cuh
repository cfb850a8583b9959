// Plan data structures shared by net.cu (schedule + inference) and net_train.cu (training).
#pragma once
#include <vector>

#include "common.cuh"
#include "conv.cuh"
#include "optim.cuh"

namespace yb {

struct Ten {          // a view of an activation: buffer id + channel slice
  int buf = -1;       // -1: network input image
  int off = 0;        // first channel inside the buffer
  int c = 0, h = 0, w = 0;
};

struct Buf {
  int h, w, ld;       // [n, h, w, ld]
  int fp32;           // detection outputs are float32
  int esz = 2;        // bytes per element: 4 (fp32), 2 (fp16 / bf16), 1 (e4m3)
  size_t offset = 0, bytes = 0;
};

struct Layer {
  yb_layer_info info;
  Ten in, out, res;   // res.buf == -2: none
  bool upsample = false, out_fp32 = false;
  int cout_pad = 0;
  int dtype = 0;      // yb_dtype of the conv's input and packed weights (e4m3 plan: fp16 for layers 0-3)
  // parameter arena offsets (bytes); w_scale: e4m3 layers' per-output-channel weight scales, fp32 [cout_pad]
  size_t w_master = 0, w_packed = 0, gamma = 0, beta = 0, mean = 0, var = 0, bias = 0, scale = 0, shift = 0, w_scale = 0;
  // prepared implicit-GEMM launch of the inference forward
  ConvLaunch fwd;
  // Cin <= 64 3x3 layers: prepared halo-tile launch (csrc/conv_halo.cu), inference forward only
  HaloLaunch halo;
  // detection heads: the same conv with the decode + NMS candidate filter fused into its epilogue (yb_net_detect)
  ConvLaunch det;
  bool det_ok = false;
  // ---- training plan (net_train.cu) ----
  size_t z_off = 0, dz_off = 0;      // raw conv output z / its gradient (activation arena); dz is zero-inserted for stride 2
  int dz_ld = 0, dz_dilated = 0, k_cout = 0;
  int dgrad_parity = 0;              // stride-2 layer whose dgrad runs as 4 parity-class convs on the plain dz
  size_t st_sum = 0, st_sqsum = 0, st_mean = 0, st_invstd = 0, st_scale = 0, st_shift = 0;   // fp32 [cout_pad] each
  size_t x_bwd = 0;                  // fp32 [2][cout_pad]: sync-BN backward exchange slab (sum dact*zhat | sum dact)
  size_t w_dgrad = 0;                // [cin_pad, k, k, k_cout] 16-bit (param arena)
  long g_w = -1, g_gamma = -1, g_beta = -1, g_bias = -1;   // float offsets into the flat gradient / velocity buffers
  ConvLaunch train;                  // training-mode forward conv: raw z + statistics (detection heads: fwd)
  // dgrad: the forward kernel on dz with flipped/transposed weights; stride-2 parity layers: one launch per class
  ConvLaunch dgrad[4];
  int num_dgrad = 0;                 // 1 | 4
  WgradLaunch wgrad;                 // weight gradient (layers >= 1; the stem's reads the step's image)
};

// the activation view t (16-bit training buffers and inference buffers of any element size)
void* ten_ptr(const yb_net* net, const Ten& t);
// conv descriptor of a tensor-core layer's inference forward (the training plan derives its own from it)
yb_conv_desc layer_desc(const yb_net* net, const Layer& L);

}  // namespace yb

struct yb_net {
  int class_num, n, h, w, dtype, training;
  std::vector<yb::Layer> layers;
  std::vector<yb::Buf> bufs;
  int fm_buf[3];
  size_t act_bytes = 0, param_bytes = 0;
  // e4m3 plan: per-buffer activation scale (value = code x scale; 1 for 16-bit / fp32 buffers), set by calibration
  std::vector<float> buf_scale;
  bool fp8_ready = false;
  uint8_t* act = nullptr;
  uint8_t* par = nullptr;
  // ---- training plan ----
  std::vector<size_t> gbuf_offset;   // gradient mirror of every 16-bit activation buffer
  size_t dfm_off[3] = {0, 0, 0};     // 16-bit [rows, 256] loss gradients of the three detection maps
  size_t stats_off = 0, stats_bytes = 0;   // per-step zeroed BN sums
  size_t xbwd_off = 0, xbwd_bytes = 0;     // sync-BN backward exchange slabs
  size_t lossws_off = 0, lossws_bytes = 0;
  size_t bnws_off = 0, bnws_bytes = 0;     // two-stage BN-backward reduction scratch (zeroed at bind)
  size_t ones_off = 0, zeros_off = 0;      // fp32 [1024] constants (param arena)
  size_t grad_off = 0, vel_off = 0; long grad_count = 0;   // flat fp32 gradient / optimizer slots (param arena)
  int opt_state_slots = 2;            // slot 1: momentum / adam m; slot 2: rmsprop mean square / adam v
  size_t opt_step_off = 0;            // int ctrl[64]: non-finite flag, updates applied, steps skipped
  size_t opt_tensors_off = 0, opt_chunks_off = 0, opt_norm_off = 0; int num_opt_tensors = 0, num_opt_chunks = 0;
  std::vector<yb::OptTensor> opt_tensors;
  std::vector<yb::OptChunk> opt_chunks;
  size_t pack_jobs_off = 0; int pack_tiles = 0;   // multi-tensor dgrad-weight repack (optim.cuh: PackJob)
  std::vector<yb::PackJob> pack_jobs;
  bool fold_dirty = false;
  float bn_eps = 1e-5f;
  // side stream of the backward pass: layer L's wgrad runs beside its dgrad (net_train.cu); created on first use
  cudaStream_t side_stream = nullptr;
  cudaEvent_t side_fork = nullptr, side_join = nullptr;
  bool side_forked = false;           // work on the side stream not yet joined
  // layered training step (yb_net_train_forward_layer ...): the feature maps the forward wrote, and the next call
  float* train_fm[3] = {nullptr, nullptr, nullptr};
  int step_slot = -1, step_replicas = 1;
  ~yb_net() {
    if (side_fork) cudaEventDestroy(side_fork);
    if (side_join) cudaEventDestroy(side_join);
    if (side_stream) cudaStreamDestroy(side_stream);
  }
};

