// Training plan: one step of train.py:105-115 on the H100 engine.
//   forward  : conv (raw z + BN batch sums in the epilogue) -> bn_finalize -> bn_act_apply
//              (model.py:30-80 with is_training=True; UPDATE_OPS moving stats, train.py:108-109)
//   loss     : yb_loss_layer x3, gradients written 16-bit into the backward GEMM operands
//   backward : per layer, last to first: bn_bwd_reduce/apply -> wgrad (wgmma) -> dgrad (forward
//              kernel on dz with flipped/transposed weights; the residual / second-consumer
//              contributions are folded into the dgrad epilogue's residual add)
//   update   : L2 + per-tensor clip_by_norm + momentum over one flat gradient buffer (which the
//              data-parallel wrapper all-reduces between backward and update).
#include <string.h>

#include <algorithm>
#include <map>

#include "net.cuh"

namespace yb {

// bn.cu: the BN kernels with the row count and the backward exchange slab exposed
int bn_stats_act_apply_n(const void* z, long z_ld, const float* sum, const float* sqsum, long count, const float* gamma,
                         const float* beta, float eps, float decay, float* moving_mean, float* moving_var, float* scale,
                         float* shift, float* save_mean, float* save_invstd, const void* res, long res_ld, void* out,
                         long out_ld, int n, int h, int w, int c, int dtype, int leaky, int upsample2x, void* stream);
int bn_bwd_reduce_x(const void* dA, long dA_ld, const void* z, long z_ld, const float* scale, const float* shift,
                    const float* save_mean, const float* save_invstd, int n, int h, int w, int c, int dtype, int leaky,
                    int upsample2x, float* dgamma, float* dbeta, void* workspace, float* xg, float* xb, void* stream);
int bn_bwd_apply_n(const void* dA, long dA_ld, const void* z, long z_ld, const float* gamma, const float* scale,
                   const float* shift, const float* save_mean, const float* save_invstd, const float* dgamma,
                   const float* dbeta, long count, int n, int h, int w, int c, int dtype, int leaky, int upsample2x,
                   int dilate2x, void* dz, long dz_ld, void* stream);

static size_t al256(size_t v) { return (v + 255) & ~size_t(255); }

// Extend the arenas computed by Builder::build() with everything training needs.
void train_layout(yb_net* net) {
  const size_t esz = 2;
  size_t o = net->act_bytes;
  // gradient mirrors of the 16-bit activation buffers
  net->gbuf_offset.assign(net->bufs.size(), 0);
  for (size_t b = 0; b < net->bufs.size(); ++b) {
    if (net->bufs[b].fp32) continue;
    net->gbuf_offset[b] = o;
    o = al256(o + net->bufs[b].bytes);
  }
  int head_i = 0;
  for (auto& L : net->layers) {
    const size_t out_rows = (size_t)net->n * L.info.out_h * L.info.out_w;
    L.k_cout = (L.info.cout + 31) / 32 * 32;
    if (L.info.has_bn) {
      L.z_off = o; o = al256(o + out_rows * L.info.cout * esz);
      L.dz_ld = L.info.cout;
      // stride-2 layers: the input gradient is computed per parity class on the plain dz (4 small convs, no zeros);
      // YB_DGRAD_S2=dilated selects the first version (one 3x3 conv over a zero-inserted dz: 4x the MMA work)
      const char* s2 = opt("YB_DGRAD_S2");
      L.dgrad_parity = (L.info.stride == 2 && !(s2 && s2[0] == 'd')) ? 1 : 0;
      L.dz_dilated = L.info.stride == 2 && !L.dgrad_parity;
      const size_t dz_rows = L.dz_dilated ? (size_t)net->n * L.info.in_h * L.info.in_w : out_rows;
      L.dz_off = o; o = al256(o + dz_rows * L.dz_ld * esz);
    } else {
      L.dz_ld = L.k_cout;                      // 255 -> 256, zero padded by the loss kernel
      L.dz_off = o; o = al256(o + out_rows * L.dz_ld * esz);
      net->dfm_off[head_i++] = L.dz_off;
    }
  }
  // per-step-zeroed BN sums, then the other per-channel scratch
  net->stats_off = o;
  for (auto& L : net->layers) {
    if (!L.info.has_bn) continue;
    L.st_sum = o; o += (size_t)L.cout_pad * 4;
    L.st_sqsum = o; o += (size_t)L.cout_pad * 4;
  }
  o = al256(o);
  net->stats_bytes = o - net->stats_off;
  // backward exchange slabs [sum dact*zhat | sum dact] of synchronised BN (padding zeroed at bind)
  net->xbwd_off = o;
  for (auto& L : net->layers) {
    if (!L.info.has_bn) continue;
    L.x_bwd = o; o += 2 * (size_t)L.cout_pad * 4;
  }
  o = al256(o);
  net->xbwd_bytes = o - net->xbwd_off;
  for (auto& L : net->layers) {
    if (!L.info.has_bn) continue;
    L.st_mean = o; o = al256(o + (size_t)L.cout_pad * 4);
    L.st_invstd = o; o = al256(o + (size_t)L.cout_pad * 4);
    L.st_scale = o; o = al256(o + (size_t)L.cout_pad * 4);
    L.st_shift = o; o = al256(o + (size_t)L.cout_pad * 4);
  }
  size_t lw = 0;
  for (int s = 0; s < 3; ++s) {
    size_t b = 0;
    const int div = 32 >> s;
    yb_loss_workspace_bytes(net->n, net->h / div, net->w / div, &b);
    lw = std::max(lw, b);
  }
  net->lossws_off = o; net->lossws_bytes = lw; o = al256(o + lw);
  yb_bn_bwd_reduce_workspace_bytes(&net->bnws_bytes);
  net->bnws_off = o; o = al256(o + net->bnws_bytes);
  net->act_bytes = o;

  // ---- parameter arena ----
  o = net->param_bytes;
  net->ones_off = o; o = al256(o + 1024 * 4);
  net->zeros_off = o; o = al256(o + 1024 * 4);
  for (auto& L : net->layers) {
    if (L.info.index == 0) continue;
    const size_t cin_pad = yb_conv_cout_pad(L.info.cin);
    L.w_dgrad = o;
    o = al256(o + cin_pad * L.info.ksize * L.info.ksize * L.k_cout * esz);
  }
  long g = 0;
  auto take = [&](long n) { long at = g; g += (n + 3) / 4 * 4; return at; };
  for (auto& L : net->layers) {
    L.g_w = take((long)L.info.cout * L.info.ksize * L.info.ksize * L.info.cin);
    if (L.info.has_bn) { L.g_gamma = take(L.info.cout); L.g_beta = take(L.info.cout); }
    else L.g_bias = take(L.info.cout);
  }
  net->grad_count = g;
  net->grad_off = o; o = al256(o + (size_t)g * 4);
  net->vel_off = o; o = al256(o + (size_t)g * 4 * net->opt_state_slots);
  // optimizer tables
  net->opt_tensors.clear(); net->opt_chunks.clear();
  const long CH = 1 << 16;
  auto add = [&](long n, int l2) {
    OptTensor t; memset(&t, 0, sizeof(t));
    t.n = n; t.l2 = l2; t.trainable = 1;
    const int id = (int)net->opt_tensors.size();
    net->opt_tensors.push_back(t);
    for (long b = 0; b < n; b += CH) { OptChunk c; c.tensor = id; c.begin = b; c.end = std::min(n, b + CH); net->opt_chunks.push_back(c); }
  };
  for (auto& L : net->layers) {
    add((long)L.info.cout * L.info.ksize * L.info.ksize * L.info.cin, 1);
    if (L.info.has_bn) { add(L.info.cout, 0); add(L.info.cout, 0); } else add(L.info.cout, 0);
  }
  net->num_opt_tensors = (int)net->opt_tensors.size();
  net->num_opt_chunks = (int)net->opt_chunks.size();
  net->opt_tensors_off = o; o = al256(o + net->opt_tensors.size() * sizeof(OptTensor));
  net->opt_chunks_off = o; o = al256(o + net->opt_chunks.size() * sizeof(OptChunk));
  net->opt_norm_off = o; o = al256(o + net->opt_tensors.size() * 4);
  net->opt_step_off = o; o = al256(o + 256);
  net->pack_jobs_off = o; o = al256(o + net->layers.size() * sizeof(PackJob));
  net->param_bytes = o;
}

static void* gten_ptr(const yb_net* net, const Ten& t) {
  return net->act + net->gbuf_offset[t.buf] + (size_t)t.off * 2;
}
static float* fpar(const yb_net* net, size_t off) { return reinterpret_cast<float*>(net->par + off); }
static float* fact(const yb_net* net, size_t off) { return reinterpret_cast<float*>(net->act + off); }
static float* gradp(const yb_net* net, long idx) { return reinterpret_cast<float*>(net->par + net->grad_off) + idx; }

__global__ void fill_f32_kernel(float* p, long n, float v) {
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) p[i] = v;
}

// Called from yb_net_bind for training plans.  Everything is enqueued on the caller's stream.  The optimizer state
// (velocity) lives in the parameter arena, which several plans of different shapes may share: binding never touches it —
// yb_net_train_reset_state() zeroes it once, when the arena is created.
int train_bind(yb_net* net, cudaStream_t st) {
  // constants (idempotent) + this plan's activation-arena scratch
  fill_f32_kernel<<<4, 256, 0, st>>>(fpar(net, net->ones_off), 1024, 1.0f);
  YB_CUDA(cudaGetLastError());
  YB_CUDA(cudaMemsetAsync(net->par + net->zeros_off, 0, 1024 * 4, st));
  YB_CUDA(cudaMemsetAsync(net->act + net->bnws_off, 0, net->bnws_bytes, st));
  YB_CUDA(cudaMemsetAsync(net->act + net->xbwd_off, 0, net->xbwd_bytes, st));
  const float* ones = fpar(net, net->ones_off);
  const float* zeros = fpar(net, net->zeros_off);
  for (auto& L : net->layers) {
    if (L.dz_dilated)
      YB_CUDA(cudaMemsetAsync(net->act + L.dz_off, 0, (size_t)net->n * L.info.in_h * L.info.in_w * L.dz_ld * 2, st));
  }
  // ---- training-mode forward convs: raw z + statistics; weight gradients ----
  for (size_t i = 1; i < net->layers.size(); ++i) {
    Layer& L = net->layers[i];
    const yb_conv_desc d = layer_desc(net, L);
    int rc = wgrad_prepare(&d, ten_ptr(net, L.in), net->act + L.dz_off, L.dz_ld, L.dz_dilated, gradp(net, L.g_w), &L.wgrad);
    if (rc) return rc;
    if (!L.info.has_bn) { L.train = L.fwd; continue; }   // detection convs run as in inference
    ConvRequest r{d};   // raw z [rows, cout]: no activation, residual or upsampling
    r.d.out_ld = L.info.cout; r.d.res_ld = 0; r.d.leaky = 0; r.d.upsample2x = 0;
    r.stats = true;
    rc = conv_prepare(r, ten_ptr(net, L.in), net->par + L.w_packed, ones, zeros, nullptr, net->act + L.z_off,
                      fact(net, L.st_sum), fact(net, L.st_sqsum), &L.train);
    if (rc) return rc;
  }
  // ---- dgrad convs + residual bookkeeping (reverse order) ----
  std::map<int, std::vector<std::pair<int, int>>> written;   // gradient buffer -> channel intervals already produced
  struct Pending { const void* ptr; long ld; };
  std::map<std::pair<int, int>, Pending> pending;            // (buf, off) -> residual pass-through source
  auto covered = [&](const Ten& t) {
    auto it = written.find(t.buf);
    if (it == written.end()) return false;
    for (auto& iv : it->second) if (iv.first <= t.off && t.off + t.c <= iv.first + iv.second) return true;
    return false;
  };
  for (int i = (int)net->layers.size() - 1; i >= 1; --i) {
    Layer& L = net->layers[i];
    // this layer's residual input receives dA(out) unchanged
    if (L.res.buf >= 0) pending[{L.res.buf, L.res.off}] = Pending{gten_ptr(net, L.out), (long)net->bufs[L.out.buf].ld};
    // dgrad: dA(in) (+)= conv_s1(dz [zero-inserted if stride 2], Wd)
    const void* res = nullptr;
    int res_ld = 0;
    auto pit = pending.find({L.in.buf, L.in.off});
    const bool cov = covered(L.in);
    if (cov && pit != pending.end()) { set_error("train plan: tensor with both a written gradient and a pending residual"); return YB_ERR_UNSUPPORTED; }
    if (cov) { res = gten_ptr(net, L.in); res_ld = net->bufs[L.in.buf].ld; }
    else if (pit != pending.end()) { res = pit->second.ptr; res_ld = (int)pit->second.ld; pending.erase(pit); }
    const yb_conv_desc fwd = layer_desc(net, L);
    void* dx = gten_ptr(net, L.in);
    int rc;
    if (L.dgrad_parity) {   // plain dz at the OUTPUT resolution
      L.num_dgrad = 4;
      rc = conv_prepare_dgrad_s2(&fwd, net->act + L.dz_off, L.dz_ld, L.k_cout, net->par + L.w_dgrad, res, res_ld, dx,
                                 fwd.in_ld, L.dgrad);
    } else {                // dz (dilated for stride 2) at the INPUT resolution
      L.num_dgrad = 1;
      ConvRequest r{fwd};
      r.d.cin = L.k_cout; r.d.cout = L.info.cin; r.d.stride = 1;
      r.d.in_ld = L.dz_ld; r.d.out_ld = fwd.in_ld; r.d.res_ld = res_ld; r.d.out_fp32 = 0; r.d.leaky = 0; r.d.upsample2x = 0;
      r.res = res != nullptr;
      rc = conv_prepare(r, net->act + L.dz_off, net->par + L.w_dgrad, ones, zeros, res, dx, nullptr, nullptr, &L.dgrad[0]);
    }
    if (rc) return rc;
    written[L.in.buf].push_back({L.in.off, L.in.c});
  }
  if (!pending.empty()) { set_error("train plan: unconsumed residual gradient"); return YB_ERR_UNSUPPORTED; }
  // ---- optimizer tables ----
  {
    size_t ti = 0;
    float* gbase = reinterpret_cast<float*>(net->par + net->grad_off);
    float* vbase = reinterpret_cast<float*>(net->par + net->vel_off);
    float* v2base = vbase + net->grad_count;
    for (auto& L : net->layers) {
      OptTensor& tw = net->opt_tensors[ti++];
      tw.w = fpar(net, L.w_master); tw.g = gbase + L.g_w; tw.v = vbase + L.g_w; tw.v2 = v2base + L.g_w; tw.w16 = net->par + L.w_packed;
      if (L.info.index == 0) tw.w16 = nullptr;     // the stem reads its fp32 master weights
      if (L.info.has_bn) {
        OptTensor& tg = net->opt_tensors[ti++];
        tg.w = fpar(net, L.gamma); tg.g = gbase + L.g_gamma; tg.v = vbase + L.g_gamma; tg.v2 = v2base + L.g_gamma; tg.w16 = nullptr;
        OptTensor& tb = net->opt_tensors[ti++];
        tb.w = fpar(net, L.beta); tb.g = gbase + L.g_beta; tb.v = vbase + L.g_beta; tb.v2 = v2base + L.g_beta; tb.w16 = nullptr;
      } else {
        OptTensor& tb = net->opt_tensors[ti++];
        tb.w = fpar(net, L.bias); tb.g = gbase + L.g_bias; tb.v = vbase + L.g_bias; tb.v2 = v2base + L.g_bias; tb.w16 = nullptr;
      }
    }
    // (pageable host source: the copies are staged before the calls return; the vectors live as long as the plan)
    YB_CUDA(cudaMemcpyAsync(net->par + net->opt_tensors_off, net->opt_tensors.data(), net->opt_tensors.size() * sizeof(OptTensor),
                            cudaMemcpyHostToDevice, st));
    YB_CUDA(cudaMemcpyAsync(net->par + net->opt_chunks_off, net->opt_chunks.data(), net->opt_chunks.size() * sizeof(OptChunk),
                            cudaMemcpyHostToDevice, st));
    // dgrad-weight repack table: every layer but the stem, one launch (pack_dgrad_all)
    net->pack_jobs.clear();
    int tile0 = 0;
    for (auto& L : net->layers) {
      if (L.info.index == 0) continue;
      PackJob j; memset(&j, 0, sizeof(j));
      j.w = fpar(net, L.w_master); j.dst = net->par + L.w_dgrad;
      j.cout = L.info.cout; j.cin = L.info.cin; j.ks = L.info.ksize; j.kco = L.k_cout;
      j.cin_pad = yb_conv_cout_pad(L.info.cin); j.s2 = L.dgrad_parity ? 1 : 0;
      j.tiles_ci = (j.cin_pad + 31) / 32; j.tiles_co = (j.kco + 127) / 128;
      j.tile0 = tile0;
      tile0 += j.ks * j.ks * j.tiles_ci * j.tiles_co;
      net->pack_jobs.push_back(j);
    }
    net->pack_tiles = tile0;
    YB_CUDA(cudaMemcpyAsync(net->par + net->pack_jobs_off, net->pack_jobs.data(), net->pack_jobs.size() * sizeof(PackJob),
                            cudaMemcpyHostToDevice, st));
  }
  return YB_OK;
}

// dgrad weights follow the master weights (after set_conv_params and after every update)
int train_refresh_dgrad_weights(yb_net* net, int layer, void* stream) {
  Layer& L = net->layers[layer];
  if (layer == 0) return YB_OK;
  if (L.dgrad_parity)
    return yb_pack_dgrad_weights_s2(fpar(net, L.w_master), L.info.cout, L.info.cin, L.k_cout, yb_conv_cout_pad(L.info.cin),
                                    net->dtype, net->par + L.w_dgrad, stream);
  return yb_pack_dgrad_weights(fpar(net, L.w_master), L.info.cout, L.info.cin, L.info.ksize, L.k_cout,
                               yb_conv_cout_pad(L.info.cin), net->dtype, net->par + L.w_dgrad, stream);
}

// ... all layers: one multi-tensor launch (YB_PACK_MT=0: the per-layer kernels)
static int refresh_all_dgrad_weights(yb_net* net, void* stream) {
  if (opt("YB_PACK_MT")[0] != '0' && !net->pack_jobs.empty())
    return pack_dgrad_all(reinterpret_cast<const PackJob*>(net->par + net->pack_jobs_off), (int)net->pack_jobs.size(),
                          net->pack_tiles, net->dtype, static_cast<cudaStream_t>(stream));
  for (size_t i = 1; i < net->layers.size(); ++i) {
    int rc = train_refresh_dgrad_weights(net, (int)i, stream);
    if (rc) return rc;
  }
  return YB_OK;
}

}  // namespace yb

using namespace yb;

namespace yb {

// ---- one training step as per-layer, two-phase steps -------------------------------------------------------------
// The fused entry points (yb_net_train_fwd_bwd / yb_net_train_backward) and the layered exports used by synchronised
// batch norm run the same helpers below.  LOCAL phases produce per-replica sums, GLOBAL phases consume them; under
// sync BN the caller all-reduces the layer's exchange slab between the two.  `replicas` multiplies the row count the
// GLOBAL math divides by (every rank runs the same n x h x w in a step); the fused path passes 1.

// forward.  LOCAL: the conv and its batch sums (layer 0 also zeroes the per-step sums and, unless forward-only, the
// flat gradient); a detection conv is done here.  GLOBAL: sums -> scale/shift (+ moving statistics) -> apply.
static int train_fwd_layer(yb_net* net, int i, int phase, const float* images, int replicas, float bn_decay,
                           float* const user_fm[3], int flags, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const bool bn_frozen = (flags & YB_TRAIN_BN_FROZEN) != 0;
  const int n = net->n, dt = net->dtype;
  const float* ones = fpar(net, net->ones_off);
  const float* zeros = fpar(net, net->zeros_off);
  Layer& L = net->layers[i];
  const long rows = (long)n * L.info.out_h * L.info.out_w;
  int rc;
  if (phase == YB_PHASE_LOCAL) {
    if (i == 0) {
      YB_CUDA(cudaMemsetAsync(net->act + net->stats_off, 0, net->stats_bytes, st));
      if (!(flags & YB_TRAIN_FORWARD_ONLY)) YB_CUDA(cudaMemsetAsync(net->par + net->grad_off, 0, (size_t)net->grad_count * 4, st));
      if (opt("YB_STEM_TRAIN")[0] != 'c') {   // warp-level tensor path, batch statistics accumulated by the same kernel
        return yb_stem_conv_fwd_tc_stats(images, fpar(net, L.w_master), ones, zeros, n, net->h, net->w, dt, 0,
                                         net->act + L.z_off, fact(net, L.st_sum), fact(net, L.st_sqsum), stream);
      }
      // YB_STEM_TRAIN=cuda: the fp32 CUDA-core stem + a column-statistics pass (the first version)
      rc = yb_stem_conv_fwd(images, fpar(net, L.w_master), ones, zeros, n, net->h, net->w, L.info.cout, dt, 0,
                            net->act + L.z_off, stream);
      if (rc) return rc;
      return yb_col_stats(net->act + L.z_off, L.info.cout, rows, L.info.cout, dt, fact(net, L.st_sum), fact(net, L.st_sqsum), stream);
    }
    ConvLaunch l = L.train;
    if (!L.info.has_bn) {
      const int which = L.out.buf == net->fm_buf[0] ? 0 : (L.out.buf == net->fm_buf[1] ? 1 : 2);
      l.p.out = user_fm[which] ? (void*)user_fm[which] : (void*)(net->act + net->bufs[L.out.buf].offset);
      net->train_fm[which] = static_cast<float*>(l.p.out);
    }
    return conv_launch(l, st);
  }
  if (!L.info.has_bn) return YB_OK;
  if (!bn_frozen) net->fold_dirty = true;
  const long count = (long)replicas * rows;
  const void* resp = L.res.buf >= 0 ? ten_ptr(net, L.res) : nullptr;
  const long res_ld = L.res.buf >= 0 ? net->bufs[L.res.buf].ld : 0;
  if (opt("YB_BN_FIN")[0] != '0') {   // statistics -> scale/shift inside the apply kernel (one launch per BN layer instead of two)
    return bn_stats_act_apply_n(net->act + L.z_off, L.info.cout, bn_frozen ? nullptr : fact(net, L.st_sum),
                                bn_frozen ? nullptr : fact(net, L.st_sqsum), count, fpar(net, L.gamma), fpar(net, L.beta),
                                net->bn_eps, bn_decay, fpar(net, L.mean), fpar(net, L.var), fact(net, L.st_scale),
                                fact(net, L.st_shift), fact(net, L.st_mean), fact(net, L.st_invstd), resp, res_ld,
                                ten_ptr(net, L.out), net->bufs[L.out.buf].ld, n, L.info.out_h, L.info.out_w,
                                L.info.cout, dt, 1, L.upsample ? 1 : 0, stream);
  }
  rc = yb_bn_finalize(bn_frozen ? nullptr : fact(net, L.st_sum), bn_frozen ? nullptr : fact(net, L.st_sqsum), count,
                      L.info.cout, fpar(net, L.gamma), fpar(net, L.beta),
                      net->bn_eps, bn_decay, fpar(net, L.mean), fpar(net, L.var), fact(net, L.st_scale),
                      fact(net, L.st_shift), fact(net, L.st_mean), fact(net, L.st_invstd), stream);
  if (rc) return rc;
  return yb_bn_act_apply(net->act + L.z_off, L.info.cout, fact(net, L.st_scale), fact(net, L.st_shift), resp, res_ld,
                         ten_ptr(net, L.out), net->bufs[L.out.buf].ld, n, L.info.out_h, L.info.out_w, L.info.cout, dt, 1,
                         L.upsample ? 1 : 0, stream);
}

// loss + d(loss)/d(feature maps) of the maps the forward wrote (loss4 accumulates; the callers zero it)
static int train_loss(yb_net* net, const float* const y_true[3], const float* anchors9x2, int use_label_smooth,
                      int use_focal_loss, float loss_scale, double* loss4, void* stream) {
  const int n = net->n;
  for (int s = 0; s < 3; ++s) {
    const int div = 32 >> s;
    int rc = yb_loss_layer(net->train_fm[s], y_true[s], n, net->h / div, net->w / div, net->h, net->w, net->class_num,
                           anchors9x2 + 2 * 3 * (2 - s), use_label_smooth, use_focal_loss, 1.0f / (float)n, loss_scale,
                           net->act + net->lossws_off, net->lossws_bytes, loss4, net->act + net->dfm_off[s], net->dtype,
                           (3 * (5 + net->class_num) + 31) / 32 * 32, stream);
    if (rc) return rc;
  }
  return YB_OK;
}

// makes `stream` wait for the wgrad side stream (no-op when nothing was forked since the last join)
static int train_join(yb_net* net, cudaStream_t st) {
  if (!net->side_forked) return YB_OK;
  YB_CUDA(cudaEventRecord(net->side_join, net->side_stream));
  YB_CUDA(cudaStreamWaitEvent(st, net->side_join, 0));
  net->side_forked = false;
  return YB_OK;
}

// backward.  LOCAL: the BN gradient sums (dgamma / dbeta; with `exchange` also into the layer's exchange slab), or the
// bias gradient of a detection conv.  GLOBAL: dz from the sums (the slab's with `exchange`), then wgrad and dgrad.
//
// Synchronised BN.  With W ranks of N images each, the loss is a mean over the local batch, so rank r's dA_r is
// W x the gradient of the global loss (mean over W*N) w.r.t. its rows.  The normalisation over all M = W*n*h*w rows
// makes the exact input gradient of the concatenated batch, for rank r's rows,
//   dz_r = gamma*invstd*(dact_r - SUM_ranks(sum dact)/M - zhat_r * SUM_ranks(sum dact*zhat)/M)
// evaluated with the global-loss dact; using the rank-local dact_r (W x that) gives W x the big-batch dz.  Everything
// below is linear in dz, so every weight gradient of rank r is W x its share of the big-batch gradient, and the
// all-reduce (sum) of the flat gradient followed by the optimizer's 1/W gives exactly the big-batch gradient.  The
// same holds for dgamma / dbeta, which therefore keep the LOCAL sums in the flat gradient.
static int train_bwd_layer(yb_net* net, int i, int phase, const float* images, int replicas, bool exchange, int flags,
                           void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const bool bn_frozen = (flags & YB_TRAIN_BN_FROZEN) != 0;
  const int n = net->n, dt = net->dtype;
  Layer& L = net->layers[i];
  const long rows = (long)n * L.info.out_h * L.info.out_w;
  float* xg = exchange && L.info.has_bn ? fact(net, L.x_bwd) : nullptr;
  float* xb = xg ? xg + L.cout_pad : nullptr;
  int rc;
  if (phase == YB_PHASE_LOCAL) {
    if (!L.info.has_bn) return yb_col_sum(net->act + L.dz_off, L.dz_ld, rows, L.info.cout, dt, gradp(net, L.g_bias), stream);
    return bn_bwd_reduce_x(gten_ptr(net, L.out), net->bufs[L.out.buf].ld, net->act + L.z_off, L.info.cout,
                           fact(net, L.st_scale), fact(net, L.st_shift), fact(net, L.st_mean), fact(net, L.st_invstd), n,
                           L.info.out_h, L.info.out_w, L.info.cout, dt, 1, L.upsample ? 1 : 0, gradp(net, L.g_gamma),
                           gradp(net, L.g_beta), net->act + net->bnws_off, xg, xb, stream);
  }
  if (L.info.has_bn) {
    // frozen BN: mean / variance are constants -> dz = gamma * invstd * dact (the batch-statistic terms vanish)
    const float* zeros = fpar(net, net->zeros_off);
    const float* sg = bn_frozen ? zeros : (xg ? xg : gradp(net, L.g_gamma));
    const float* sb = bn_frozen ? zeros : (xb ? xb : gradp(net, L.g_beta));
    rc = bn_bwd_apply_n(gten_ptr(net, L.out), net->bufs[L.out.buf].ld, net->act + L.z_off, L.info.cout, fpar(net, L.gamma),
                        fact(net, L.st_scale), fact(net, L.st_shift), fact(net, L.st_mean), fact(net, L.st_invstd), sg, sb,
                        (long)replicas * rows, n, L.info.out_h, L.info.out_w, L.info.cout, dt, 1, L.upsample ? 1 : 0,
                        L.dz_dilated, net->act + L.dz_off, L.dz_ld, stream);
    if (rc) return rc;
  }
  if (i == 0) return yb_stem_conv_wgrad(images, net->act + L.dz_off, dt, n, net->h, net->w, gradp(net, L.g_w), stream);
  // Layer L's weight gradient and input gradient both only read dz_L: the wgrad goes to a side stream and runs beside
  // the dgrad (and the next layer's BN backward).  Both kernels own a whole SM per CTA, so the gain is in the tails:
  // the SMs a finishing kernel frees — and the ~15 us every wgrad CTA spends flushing fp32 atomics at its end — are
  // picked up by the other kernel's CTAs instead of idling until the launch boundary.  dz_L and the forward activations
  // are never rewritten during the backward (one buffer per layer); train_join orders the side stream before whatever
  // the caller enqueues next (all-reduce of a finished layer range, optimizer, next step's gradient memset).
  void* wstream = stream;
  if (opt("YB_WGRAD_STREAM")[0] != '0') {
    if (net->side_stream == nullptr) {
      YB_CUDA(cudaStreamCreateWithFlags(&net->side_stream, cudaStreamNonBlocking));
      YB_CUDA(cudaEventCreateWithFlags(&net->side_fork, cudaEventDisableTiming));
      YB_CUDA(cudaEventCreateWithFlags(&net->side_join, cudaEventDisableTiming));
    }
    YB_CUDA(cudaEventRecord(net->side_fork, st));
    YB_CUDA(cudaStreamWaitEvent(net->side_stream, net->side_fork, 0));
    wstream = net->side_stream;
    net->side_forked = true;
  }
  rc = wgrad_launch(L.wgrad, static_cast<cudaStream_t>(wstream));
  if (rc) return rc;
  for (int c = 0; c < L.num_dgrad; ++c) {
    rc = conv_launch(L.dgrad[c], st);
    if (rc) return rc;
  }
  return YB_OK;
}

// Position of (layer, phase) in the layered step: forward 0..L-1 (LOCAL, GLOBAL each), the loss, backward L-1..0.
static int fwd_slot(int layer, int phase) { return 2 * layer + phase; }
static int loss_slot(const yb_net* net) { return 2 * (int)net->layers.size(); }
static int bwd_slot(const yb_net* net, int layer, int phase) {
  return loss_slot(net) + 1 + 2 * ((int)net->layers.size() - 1 - layer) + phase;
}
static const char* slot_name(const yb_net* net, int s, char* buf, size_t len) {
  const int nl = (int)net->layers.size();
  if (s < 0) snprintf(buf, len, "forward layer 0 LOCAL (no step in progress)");
  else if (s < loss_slot(net)) snprintf(buf, len, "forward layer %d %s", s / 2, s % 2 ? "GLOBAL" : "LOCAL");
  else if (s == loss_slot(net)) snprintf(buf, len, "the loss");
  else if (s < bwd_slot(net, 0, 1) + 1) {
    const int k = s - loss_slot(net) - 1;
    snprintf(buf, len, "backward layer %d %s", nl - 1 - k / 2, k % 2 ? "GLOBAL" : "LOCAL");
  } else snprintf(buf, len, "forward layer 0 LOCAL (the step is complete)");
  return buf;
}
// Host-side order check: a step starts at forward layer 0 LOCAL (always accepted) and every other call must be the
// next one.  A failed or out-of-order call leaves the step unfinished; starting again at layer 0 recovers.
static int check_slot(yb_net* net, const char* what, int s, int replicas) {
  const bool start = s == 0;
  if (!start && s != net->step_slot) {
    char want[96], got[96];
    set_error("%s: out of order: called for %s, expected %s", what, slot_name(net, s, got, sizeof(got)),
              slot_name(net, net->step_slot, want, sizeof(want)));
    return YB_ERR_INVALID_ARGUMENT;
  }
  if (!start && replicas != net->step_replicas) {
    set_error("%s: bn_replicas %d differs from the %d this step started with", what, replicas, net->step_replicas);
    return YB_ERR_INVALID_ARGUMENT;
  }
  return YB_OK;
}
static int advance(yb_net* net, int s, int replicas, int rc) {
  net->step_slot = rc == YB_OK ? s + 1 : -1;
  net->step_replicas = replicas;
  return rc;
}

}  // namespace yb

extern "C" int yb_net_train_fwd_bwd(yb_net* net, const float* images, const float* y_true_1, const float* y_true_2,
                                    const float* y_true_3, const float* anchors9x2, int use_label_smooth,
                                    int use_focal_loss, float bn_decay, float loss_scale, float* fm1, float* fm2,
                                    float* fm3, double* loss4, int flags, void* stream) {
  const int forward_only = flags & YB_TRAIN_FORWARD_ONLY;
  YB_REQUIRE(net && net->training && net->act && net->par, "train_fwd_bwd: not a bound training plan");
  YB_REQUIRE(images, "train_fwd_bwd: null images");
  YB_REQUIRE(forward_only || (y_true_1 && y_true_2 && y_true_3 && anchors9x2 && loss4), "train_fwd_bwd: null pointer");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  float* user_fm[3] = {fm1, fm2, fm3};
  const float* y_true[3] = {y_true_1, y_true_2, y_true_3};
  int rc;
  net->step_slot = -1;
  if (!forward_only) YB_CUDA(cudaMemsetAsync(loss4, 0, 4 * sizeof(double), st));
  // ------------------------------------------------ forward (is_training=True)
  for (int i = 0; i < (int)net->layers.size(); ++i) {
    for (int ph = YB_PHASE_LOCAL; ph <= YB_PHASE_GLOBAL; ++ph) {
      rc = train_fwd_layer(net, i, ph, images, 1, bn_decay, user_fm, flags, stream);
      if (rc) return rc;
    }
  }
  if (forward_only) return YB_OK;
  // ------------------------------------------------ loss + d(loss)/d(feature maps)
  rc = train_loss(net, y_true, anchors9x2, use_label_smooth, use_focal_loss, loss_scale, loss4, stream);
  if (rc) return rc;
  if (flags & YB_TRAIN_NO_BACKWARD) return YB_OK;
  return yb_net_train_backward(net, images, 0, (int)net->layers.size() - 1, flags, stream);
}

// Backward of layers last_layer .. first_layer (descending), after yb_net_train_fwd_bwd(..., YB_TRAIN_NO_BACKWARD):
// lets a data-parallel caller all-reduce the finished head-side gradient buckets while the backbone is still running.
extern "C" int yb_net_train_backward(yb_net* net, const float* images, int first_layer, int last_layer, int flags,
                                     void* stream) {
  YB_REQUIRE(net && net->training && net->act && net->par && images, "train_backward: not a bound training plan");
  YB_REQUIRE(first_layer >= 0 && first_layer <= last_layer && last_layer < (int)net->layers.size(), "train_backward: bad layer range");
  net->step_slot = -1;
  for (int i = last_layer; i >= first_layer; --i) {
    for (int ph = YB_PHASE_LOCAL; ph <= YB_PHASE_GLOBAL; ++ph) {
      int rc = train_bwd_layer(net, i, ph, images, 1, false, flags, stream);
      if (rc) return rc;
    }
  }
  return train_join(net, static_cast<cudaStream_t>(stream));
}

extern "C" int yb_net_train_forward_layer(yb_net* net, const float* images, int layer, int phase, int bn_replicas,
                                          float bn_decay, float* fm1, float* fm2, float* fm3, int flags, void* stream) {
  YB_REQUIRE(net && net->training && net->act && net->par && images, "train_forward_layer: not a bound training plan");
  YB_REQUIRE(layer >= 0 && layer < (int)net->layers.size() && (phase == YB_PHASE_LOCAL || phase == YB_PHASE_GLOBAL),
             "train_forward_layer: bad layer or phase");
  YB_REQUIRE(bn_replicas >= 1, "train_forward_layer: bn_replicas must be >= 1");
  const int s = fwd_slot(layer, phase);
  int rc = check_slot(net, "train_forward_layer", s, bn_replicas);
  if (rc) return rc;
  float* user_fm[3] = {fm1, fm2, fm3};
  return advance(net, s, bn_replicas, train_fwd_layer(net, layer, phase, images, bn_replicas, bn_decay, user_fm, flags, stream));
}

extern "C" int yb_net_train_loss(yb_net* net, const float* y_true_1, const float* y_true_2, const float* y_true_3,
                                 const float* anchors9x2, int use_label_smooth, int use_focal_loss, float loss_scale,
                                 double* loss4, void* stream) {
  YB_REQUIRE(net && net->training && net->act && net->par, "train_loss: not a bound training plan");
  YB_REQUIRE(y_true_1 && y_true_2 && y_true_3 && anchors9x2 && loss4, "train_loss: null pointer");
  const int s = loss_slot(net);
  int rc = check_slot(net, "train_loss", s, net->step_replicas);
  if (rc) return rc;
  YB_CUDA(cudaMemsetAsync(loss4, 0, 4 * sizeof(double), static_cast<cudaStream_t>(stream)));
  const float* y_true[3] = {y_true_1, y_true_2, y_true_3};
  return advance(net, s, net->step_replicas,
                 train_loss(net, y_true, anchors9x2, use_label_smooth, use_focal_loss, loss_scale, loss4, stream));
}

extern "C" int yb_net_train_backward_layer(yb_net* net, const float* images, int layer, int phase, int bn_replicas,
                                           int flags, void* stream) {
  YB_REQUIRE(net && net->training && net->act && net->par && images, "train_backward_layer: not a bound training plan");
  YB_REQUIRE(layer >= 0 && layer < (int)net->layers.size() && (phase == YB_PHASE_LOCAL || phase == YB_PHASE_GLOBAL),
             "train_backward_layer: bad layer or phase");
  YB_REQUIRE(bn_replicas >= 1, "train_backward_layer: bn_replicas must be >= 1");
  const int s = bwd_slot(net, layer, phase);
  int rc = check_slot(net, "train_backward_layer", s, bn_replicas);
  if (rc) return rc;
  return advance(net, s, bn_replicas, train_bwd_layer(net, layer, phase, images, bn_replicas, true, flags, stream));
}

extern "C" int yb_net_train_join(yb_net* net, void* stream) {
  YB_REQUIRE(net && net->training, "train_join: not a training plan");
  return train_join(net, static_cast<cudaStream_t>(stream));
}

extern "C" int yb_net_bn_exchange_buffer(yb_net* net, int layer, int backward, float** ptr, size_t* count) {
  YB_REQUIRE(net && net->training && net->act && ptr && count && layer >= 0 && layer < (int)net->layers.size(),
             "bn_exchange_buffer: bad argument");
  const Layer& L = net->layers[layer];
  YB_REQUIRE(L.info.has_bn, "bn_exchange_buffer: layer %d has no batch norm", layer);
  *ptr = fact(net, backward ? L.x_bwd : L.st_sum);   // forward: st_sum and st_sqsum are adjacent
  *count = 2 * (size_t)L.cout_pad;
  return YB_OK;
}

extern "C" int yb_net_bn_batch_stats(yb_net* net, int layer, float** mean, float** invstd, float** scale,
                                     float** shift) {
  YB_REQUIRE(net && net->training && layer >= 0 && layer < (int)net->layers.size(), "bn_batch_stats: bad argument");
  const Layer& L = net->layers[layer];
  YB_REQUIRE(L.info.has_bn, "bn_batch_stats: layer %d has no batch norm", layer);
  YB_REQUIRE(net->act, "bn_batch_stats: not a bound training plan");
  if (mean) *mean = fact(net, L.st_mean);
  if (invstd) *invstd = fact(net, L.st_invstd);
  if (scale) *scale = fact(net, L.st_scale);
  if (shift) *shift = fact(net, L.st_shift);
  return YB_OK;
}

extern "C" int yb_net_train_reset_state(yb_net* net, int optimizer_kind, void* stream) {
  YB_REQUIRE(net && net->training && net->par, "train_reset_state: not a bound training plan");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  YB_CUDA(cudaMemsetAsync(net->par + net->vel_off, 0, (size_t)net->grad_count * 4 * net->opt_state_slots, st));
  if (optimizer_kind == YB_OPT_RMSPROP) {       // [TF] RMSPropOptimizer creates its `rms` slot with ones
    fill_f32_kernel<<<num_sms() * 4, 256, 0, st>>>(reinterpret_cast<float*>(net->par + net->vel_off) + net->grad_count,
                                                   net->grad_count, 1.0f);
    YB_CUDA(cudaGetLastError());
  }
  YB_CUDA(cudaMemsetAsync(net->par + net->grad_off, 0, (size_t)net->grad_count * 4, st));
  YB_CUDA(cudaMemsetAsync(net->par + net->opt_step_off, 0, 256, st));
  return YB_OK;
}

extern "C" int yb_net_opt_state(yb_net* net, float** slots, size_t* count_per_slot, int* num_slots, int** ctrl) {
  YB_REQUIRE(net && net->training && net->par, "opt_state: not a bound training plan");
  if (slots) *slots = reinterpret_cast<float*>(net->par + net->vel_off);
  if (count_per_slot) *count_per_slot = (size_t)net->grad_count;
  if (num_slots) *num_slots = net->opt_state_slots;
  if (ctrl) *ctrl = reinterpret_cast<int*>(net->par + net->opt_step_off);
  return YB_OK;
}

extern "C" int yb_net_opt_norms(yb_net* net, float** sqnorm, int* count) {
  YB_REQUIRE(net && net->training && net->par && sqnorm && count, "opt_norms: not a bound training plan");
  *sqnorm = fpar(net, net->opt_norm_off);
  *count = net->num_opt_tensors;
  return YB_OK;
}

// train.py:81 `update_part`: restrict the update to some convs (their weights, gamma/beta or bias)
extern "C" int yb_net_set_trainable(yb_net* net, int layer, int trainable, void* stream) {
  YB_REQUIRE(net && net->training && net->par && layer >= 0 && layer < (int)net->layers.size(), "set_trainable: bad argument");
  size_t ti = 0;
  for (int i = 0; i < layer; ++i) ti += net->layers[i].info.has_bn ? 3 : 2;
  const int cnt = net->layers[layer].info.has_bn ? 3 : 2;
  for (int j = 0; j < cnt; ++j) net->opt_tensors[ti + j].trainable = trainable ? 1 : 0;
  YB_CUDA(cudaMemcpyAsync(net->par + net->opt_tensors_off + ti * sizeof(OptTensor), &net->opt_tensors[ti], cnt * sizeof(OptTensor),
                          cudaMemcpyHostToDevice, static_cast<cudaStream_t>(stream)));
  return YB_OK;
}

extern "C" int yb_net_train_refresh_dgrad(yb_net* net, void* stream) {
  YB_REQUIRE(net && net->training && net->par, "train_refresh_dgrad: not a bound training plan");
  return refresh_all_dgrad_weights(net, stream);
}

extern "C" int yb_net_grad_buffer(yb_net* net, float** ptr, size_t* count) {
  YB_REQUIRE(net && net->training && net->par && ptr && count, "grad_buffer: not a bound training plan");
  *ptr = reinterpret_cast<float*>(net->par + net->grad_off);
  *count = (size_t)net->grad_count;
  return YB_OK;
}

// flat-gradient slice of layers [first_layer, last_layer] (contiguous: the buffer is laid out in creation order)
extern "C" int yb_net_grad_range(yb_net* net, int first_layer, int last_layer, float** ptr, size_t* count) {
  YB_REQUIRE(net && net->training && net->par && ptr && count, "grad_range: not a bound training plan");
  YB_REQUIRE(first_layer >= 0 && first_layer <= last_layer && last_layer < (int)net->layers.size(), "grad_range: bad layer range");
  const long lo = net->layers[first_layer].g_w;
  const long hi = last_layer + 1 < (int)net->layers.size() ? net->layers[last_layer + 1].g_w : net->grad_count;
  *ptr = reinterpret_cast<float*>(net->par + net->grad_off) + lo;
  *count = (size_t)(hi - lo);
  return YB_OK;
}

extern "C" int yb_net_train_update(yb_net* net, const yb_optimizer* opt, void* stream) {
  YB_REQUIRE(net && net->training && net->par && opt, "train_update: not a bound training plan");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int rc = opt_step(reinterpret_cast<const OptTensor*>(net->par + net->opt_tensors_off),
                    reinterpret_cast<const OptChunk*>(net->par + net->opt_chunks_off), net->num_opt_tensors,
                    net->num_opt_chunks, fpar(net, net->opt_norm_off), reinterpret_cast<int*>(net->par + net->opt_step_off),
                    net->dtype, *opt, st);
  if (rc) return rc;
  rc = refresh_all_dgrad_weights(net, stream);
  if (rc) return rc;
  net->fold_dirty = true;
  return YB_OK;
}

extern "C" int yb_net_get_conv_params(yb_net* net, int layer, float** w_ohwi, float** gamma, float** beta,
                                      float** mean, float** var, float** bias) {
  YB_REQUIRE(net && net->par && layer >= 0 && layer < (int)net->layers.size(), "get_conv_params: bad argument");
  Layer& L = net->layers[layer];
  if (w_ohwi) *w_ohwi = fpar(net, L.w_master);
  if (gamma) *gamma = L.info.has_bn ? fpar(net, L.gamma) : nullptr;
  if (beta) *beta = L.info.has_bn ? fpar(net, L.beta) : nullptr;
  if (mean) *mean = L.info.has_bn ? fpar(net, L.mean) : nullptr;
  if (var) *var = L.info.has_bn ? fpar(net, L.var) : nullptr;
  if (bias) *bias = L.info.has_bn ? nullptr : fpar(net, L.bias);
  return YB_OK;
}

extern "C" int yb_net_layer_grad(yb_net* net, int layer, float** dw, float** dgamma, float** dbeta, float** dbias) {
  YB_REQUIRE(net && net->training && net->par && layer >= 0 && layer < (int)net->layers.size(), "layer_grad: bad argument");
  Layer& L = net->layers[layer];
  if (dw) *dw = gradp(net, L.g_w);
  if (dgamma) *dgamma = L.info.has_bn ? gradp(net, L.g_gamma) : nullptr;
  if (dbeta) *dbeta = L.info.has_bn ? gradp(net, L.g_beta) : nullptr;
  if (dbias) *dbias = L.info.has_bn ? nullptr : gradp(net, L.g_bias);
  return YB_OK;
}

extern "C" int yb_net_train_buffer(yb_net* net, int layer, int which, void** ptr, int* ld, int* rows_h, int* rows_w) {
  YB_REQUIRE(net && net->training && net->act && layer >= 0 && layer < (int)net->layers.size() && ptr && ld,
             "train_buffer: bad argument");
  Layer& L = net->layers[layer];
  int h = L.info.out_h, w = L.info.out_w;
  switch (which) {
    case 0: YB_REQUIRE(L.info.has_bn, "train_buffer: no z for detection convs"); *ptr = net->act + L.z_off; *ld = L.info.cout; break;
    case 1: *ptr = net->act + L.dz_off; *ld = L.dz_ld; if (L.dz_dilated) { h = L.info.in_h; w = L.info.in_w; } break;
    case 2: YB_REQUIRE(L.info.has_bn, "train_buffer: no dA for detection convs"); *ptr = gten_ptr(net, L.out); *ld = net->bufs[L.out.buf].ld;
            if (L.upsample) { h *= 2; w *= 2; } break;
    case 3: YB_REQUIRE(layer > 0, "train_buffer: layer 0 reads the image"); *ptr = ten_ptr(net, L.in); *ld = net->bufs[L.in.buf].ld;
            h = L.info.in_h; w = L.info.in_w; break;
    case 4: YB_REQUIRE(layer > 0 && net->par, "train_buffer: the stem has no dgrad weights");   // [cin_pad * k * k][k_cout], 16-bit
            *ptr = net->par + L.w_dgrad; *ld = L.k_cout; h = yb_conv_cout_pad(L.info.cin); w = L.info.ksize * L.info.ksize; break;
    case 5: YB_REQUIRE(layer > 0, "train_buffer: the stem has no dgrad, so no input gradient");   // what the dgrad writes
            *ptr = gten_ptr(net, L.in); *ld = net->bufs[L.in.buf].ld; h = L.info.in_h; w = L.info.in_w; break;
    case 6: YB_REQUIRE(layer > 0 && net->par, "train_buffer: the stem reads its fp32 master weights");   // [cout_pad][k * k * cin]
            *ptr = net->par + L.w_packed; *ld = L.info.ksize * L.info.ksize * L.info.cin; h = L.cout_pad; w = 1; break;
    default: set_error("train_buffer: which must be 0..6"); return YB_ERR_INVALID_ARGUMENT;
  }
  if (rows_h) *rows_h = h;
  if (rows_w) *rows_w = w;
  return YB_OK;
}
