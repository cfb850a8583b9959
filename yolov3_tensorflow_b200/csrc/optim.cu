// Training-step tail (train.py:78,113-115; utils/misc_utils.py:151-161): L2 regulariser on the
// conv weights (slim.l2_regularizer: grad += wd*w), per-tensor tf.clip_by_norm(g, clip), then the
// optimizer chosen by config_optimizer — momentum (the default), rmsprop, adam or sgd with
// TensorFlow 1.x's update rules — plus the refresh of the 16-bit compute copy of every conv weight:
// all 222 trainable tensors in two multi-tensor launches driven by a device-side chunk table.
// A step whose gradient contains a non-finite value (fp16 storage with loss scaling) is skipped as a whole.
#include "common.cuh"
#include "optim.cuh"

namespace yb {

__global__ void __launch_bounds__(256)
opt_norm_kernel(const OptTensor* __restrict__ tensors, const OptChunk* __restrict__ chunks, int num_chunks,
                float grad_scale, float weight_decay, float* __restrict__ sqnorm, int* __restrict__ ctrl) {
  __shared__ float s_red[8];
  for (int ci = blockIdx.x; ci < num_chunks; ci += gridDim.x) {
    const OptChunk ch = chunks[ci];
    const OptTensor t = tensors[ch.tensor];
    if (!t.trainable) continue;
    const float wd = t.l2 ? weight_decay : 0.f;
    float acc = 0.f;
    for (long i = ch.begin + threadIdx.x; i < ch.end; i += 256) {
      const float g = t.g[i] * grad_scale + wd * t.w[i];
      acc += g * g;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
      float s = 0.f;
      for (int w = 0; w < 8; ++w) s += s_red[w];
      if (!isfinite(s)) atomicOr(ctrl, 1);
      atomicAdd(sqnorm + ch.tensor, s);
    }
    __syncthreads();
  }
}

template <typename T, int KIND>
__global__ void __launch_bounds__(256)
opt_update_kernel(const OptTensor* __restrict__ tensors, const OptChunk* __restrict__ chunks, int num_chunks,
                  const yb_optimizer o, const float* __restrict__ sqnorm, const int* __restrict__ ctrl) {
  if (ctrl[0]) return;                                                      // non-finite gradient: skip the step
  float lr = o.lr;
  if (KIND == YB_OPT_ADAM) {                                                // [TF] AdamOptimizer: lr_t = lr*sqrt(1-b2^t)/(1-b1^t)
    const float t = (float)(ctrl[1] + 1);
    lr = o.lr * sqrtf(1.f - powf(o.beta2, t)) / (1.f - powf(o.beta1, t));
  }
  for (int ci = blockIdx.x; ci < num_chunks; ci += gridDim.x) {
    const OptChunk ch = chunks[ci];
    const OptTensor t = tensors[ch.tensor];
    if (!t.trainable) continue;
    const float wd = t.l2 ? o.weight_decay : 0.f;
    const float nrm = sqrtf(sqnorm[ch.tensor]);
    const float cs = o.clip_norm > 0.f ? o.clip_norm / fmaxf(nrm, o.clip_norm) : 1.f;   // tf.clip_by_norm
    T* w16 = static_cast<T*>(t.w16);
    for (long i = ch.begin + threadIdx.x; i < ch.end; i += 256) {
      const float w = t.w[i];
      const float g = (t.g[i] * o.grad_scale + wd * w) * cs;
      float nw;
      if (KIND == YB_OPT_SGD) {                                             // [TF] GradientDescentOptimizer
        nw = w - lr * g;
      } else if (KIND == YB_OPT_MOMENTUM) {                                 // [TF] MomentumOptimizer, no Nesterov
        const float v = o.momentum * t.v[i] + g;
        t.v[i] = v;
        nw = w - lr * v;
      } else if (KIND == YB_OPT_RMSPROP) {                                  // [TF] RMSPropOptimizer (not centered)
        const float ms = o.decay * t.v2[i] + (1.f - o.decay) * g * g;
        const float mom = o.momentum * t.v[i] + lr * g * rsqrtf(ms + o.epsilon);
        t.v2[i] = ms;
        t.v[i] = mom;
        nw = w - mom;
      } else {                                                              // [TF] AdamOptimizer
        const float m = o.beta1 * t.v[i] + (1.f - o.beta1) * g;
        const float v = o.beta2 * t.v2[i] + (1.f - o.beta2) * g * g;
        t.v[i] = m;
        t.v2[i] = v;
        nw = w - lr * m / (sqrtf(v) + o.epsilon);
      }
      t.w[i] = nw;
      if (w16) w16[i] = static_cast<T>(nw);
    }
  }
}

__global__ void opt_finish_kernel(int* ctrl) {
  if (ctrl[0]) ctrl[2] += 1; else ctrl[1] += 1;
  ctrl[0] = 0;
}

int opt_step(const OptTensor* tensors, const OptChunk* chunks, int num_tensors, int num_chunks, float* sqnorm, int* ctrl,
             int dtype, const yb_optimizer& o, cudaStream_t st) {
  YB_REQUIRE(o.kind >= YB_OPT_SGD && o.kind <= YB_OPT_ADAM, "optimizer: unsupported kind %d (utils/misc_utils.py:151-161)", o.kind);
  YB_CUDA(cudaMemsetAsync(sqnorm, 0, sizeof(float) * num_tensors, st));
  const int grid = num_chunks < num_sms() * 8 ? num_chunks : num_sms() * 8;
  opt_norm_kernel<<<grid, 256, 0, st>>>(tensors, chunks, num_chunks, o.grad_scale, o.weight_decay, sqnorm, ctrl);
  YB_CUDA(cudaGetLastError());
#define YB_OPT_LAUNCH(T)                                                                                         \
  switch (o.kind) {                                                                                              \
    case YB_OPT_SGD: opt_update_kernel<T, YB_OPT_SGD><<<grid, 256, 0, st>>>(tensors, chunks, num_chunks, o, sqnorm, ctrl); break;           \
    case YB_OPT_MOMENTUM: opt_update_kernel<T, YB_OPT_MOMENTUM><<<grid, 256, 0, st>>>(tensors, chunks, num_chunks, o, sqnorm, ctrl); break; \
    case YB_OPT_RMSPROP: opt_update_kernel<T, YB_OPT_RMSPROP><<<grid, 256, 0, st>>>(tensors, chunks, num_chunks, o, sqnorm, ctrl); break;   \
    default: opt_update_kernel<T, YB_OPT_ADAM><<<grid, 256, 0, st>>>(tensors, chunks, num_chunks, o, sqnorm, ctrl); break;                  \
  }
  if (dtype == YB_BF16) { YB_OPT_LAUNCH(__nv_bfloat16) } else { YB_OPT_LAUNCH(__half) }
#undef YB_OPT_LAUNCH
  YB_CUDA(cudaGetLastError());
  opt_finish_kernel<<<1, 1, 0, st>>>(ctrl);
  YB_CUDA(cudaGetLastError());
  return YB_OK;
}

// dgrad weights: Wd[ci][r'][s'][co] = W[co][k-1-r'][k-1-s'][ci]  (flip + transpose), K padded to kco
template <typename T>
__global__ void pack_dgrad_weights_kernel(const float* __restrict__ w, int cout, int cin, int ks, int kco, int cin_pad,
                                          T* __restrict__ dst) {
  const long total = (long)cin_pad * ks * ks * kco;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int co = i % kco;
    const int s = (i / kco) % ks;
    const int r = (i / ((long)kco * ks)) % ks;
    const int ci = i / ((long)kco * ks * ks);
    float v = 0.f;
    if (co < cout && ci < cin) v = w[(((long)co * ks + (ks - 1 - r)) * ks + (ks - 1 - s)) * cin + ci];
    dst[i] = static_cast<T>(v);
  }
}

// dgrad weights of a 3x3 stride-2 conv (pad 1 + VALID, utils/layer_utils.py:17-27), split by the parity (a, b) of the
// input-gradient pixel (2i + a, 2j + b):  dx[2i+a, 2j+b] = sum over the (1+a) x (1+b) window taps (th, tw) of
//   dz[i + th, j + tw] * W[co][r][s][ci],   r = a ? (th ? 0 : 2) : 1,   s = b ? (tw ? 0 : 2) : 1.
// Four matrices [cin_pad][(1+a)(1+b) * kco] are stored back to back (class c = 2a + b at element offset
// cin_pad * kco * {0, 1, 3, 5}[c]); together they hold the 9 taps exactly once.
template <typename T>
__global__ void pack_dgrad_s2_kernel(const float* __restrict__ w, int cout, int cin, int kco, int cin_pad,
                                     T* __restrict__ dst) {
  const long per = (long)cin_pad * kco;
  const long total = 9 * per;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int cls = i < per ? 0 : (i < 3 * per ? 1 : (i < 5 * per ? 2 : 3));
    const long base = cls == 0 ? 0 : (cls == 1 ? per : (cls == 2 ? 3 * per : 5 * per));
    const int a = cls >> 1, b = cls & 1;
    const int kw = 1 + b, taps = (1 + a) * kw;
    const long j = i - base;                       // index inside [cin_pad][taps][kco]
    const int co = j % kco;
    const int tap = (j / kco) % taps;
    const int ci = j / ((long)kco * taps);
    const int th = tap / kw, tw = tap - th * kw;
    const int r = a ? (th ? 0 : 2) : 1;
    const int s2 = b ? (tw ? 0 : 2) : 1;
    float v = 0.f;
    if (co < cout && ci < cin) v = w[(((long)co * 3 + r) * 3 + s2) * cin + ci];
    dst[i] = static_cast<T>(v);
  }
}

// All layers in one launch (PackJob, optim.cuh).  The per-layer kernels above walk the DESTINATION linearly, so
// consecutive threads read the masters with a stride of ks*ks*cin floats (one 32-byte sector per element) and every
// layer pays its own launch (74 launches per training step for 370 MB of traffic).
template <typename T>
__global__ void __launch_bounds__(256) pack_dgrad_multi_kernel(const PackJob* __restrict__ jobs, int num_jobs) {
  __shared__ float tile[32][33];
  const int b = blockIdx.x;
  int lo = 0, hi = num_jobs - 1;
  while (lo < hi) {             // last job whose first tile is <= b (uniform over the block)
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(&jobs[mid].tile0) <= b) lo = mid; else hi = mid - 1;
  }
  const PackJob j = jobs[lo];
  int t = b - j.tile0;
  const int tco = t % j.tiles_co; t /= j.tiles_co;
  const int tci = t % j.tiles_ci;
  const int tap = t / j.tiles_ci;                          // SOURCE tap (kr, kc)
  const int kr = tap / j.ks, kc = tap - kr * j.ks;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int ci0 = tci * 32;
  long base = 0;
  int taps = j.ks * j.ks, dtap = (j.ks - 1 - kr) * j.ks + (j.ks - 1 - kc);
  if (j.s2) {                                              // parity classes (pack_dgrad_s2_kernel): invert r(a, th), s(b, tw)
    const int a = kr != 1, bb = kc != 1;
    const int th = (a && kr == 0) ? 1 : 0, tw = (bb && kc == 0) ? 1 : 0;
    const int kw = 1 + bb, cls = 2 * a + bb;
    taps = (1 + a) * kw;
    dtap = th * kw + tw;
    base = (long)j.cin_pad * j.kco * (cls == 0 ? 0 : (cls == 1 ? 1 : (cls == 2 ? 3 : 5)));
  }
  T* dst = static_cast<T*>(j.dst);
  for (int sub = 0; sub < 4; ++sub) {
    const int co0 = (tco * 4 + sub) * 32;
    if (co0 >= j.kco) break;
#pragma unroll
    for (int r = ty; r < 32; r += 8) {
      const int co = co0 + r, ci = ci0 + tx;
      float v = 0.f;
      if (co < j.cout && ci < j.cin) v = __ldg(j.w + (((long)co * j.ks + kr) * j.ks + kc) * j.cin + ci);
      tile[r][tx] = v;
    }
    __syncthreads();
#pragma unroll
    for (int r = ty; r < 32; r += 8) {
      const int ci = ci0 + r, co = co0 + tx;
      if (ci < j.cin_pad && co < j.kco) dst[base + ((long)ci * taps + dtap) * j.kco + co] = static_cast<T>(tile[tx][r]);
    }
    __syncthreads();
  }
}

int pack_dgrad_all(const PackJob* jobs, int num_jobs, int total_tiles, int dtype, cudaStream_t st) {
  if (num_jobs <= 0 || total_tiles <= 0) return YB_OK;
  if (dtype == YB_F16) pack_dgrad_multi_kernel<__half><<<total_tiles, 256, 0, st>>>(jobs, num_jobs);
  else if (dtype == YB_BF16) pack_dgrad_multi_kernel<__nv_bfloat16><<<total_tiles, 256, 0, st>>>(jobs, num_jobs);
  else { set_error("pack_dgrad_all: bad dtype"); return YB_ERR_UNSUPPORTED; }
  YB_CUDA(cudaGetLastError());
  return YB_OK;
}

}  // namespace yb

using namespace yb;

extern "C" int yb_pack_dgrad_weights_s2(const float* w_ohwi, int cout, int cin, int k_cout, int cin_pad, int dtype,
                                        void* dst, void* stream) {
  YB_REQUIRE(w_ohwi && dst && cout > 0 && cin > 0 && k_cout >= cout && cin_pad >= cin, "pack_dgrad_s2: bad argument");
  const long total = 9L * cin_pad * k_cout;
  const int grid = (int)((total + 255) / 256 < 148L * 16 ? (total + 255) / 256 : 148L * 16);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (dtype == YB_F16)
    pack_dgrad_s2_kernel<__half><<<grid, 256, 0, st>>>(w_ohwi, cout, cin, k_cout, cin_pad, (__half*)dst);
  else if (dtype == YB_BF16)
    pack_dgrad_s2_kernel<__nv_bfloat16><<<grid, 256, 0, st>>>(w_ohwi, cout, cin, k_cout, cin_pad, (__nv_bfloat16*)dst);
  else { set_error("pack_dgrad_s2: bad dtype"); return YB_ERR_UNSUPPORTED; }
  YB_CUDA(cudaGetLastError());
  return YB_OK;
}

extern "C" int yb_pack_dgrad_weights(const float* w_ohwi, int cout, int cin, int ksize, int k_cout, int cin_pad,
                                     int dtype, void* dst, void* stream) {
  YB_REQUIRE(w_ohwi && dst && cout > 0 && cin > 0 && k_cout >= cout && cin_pad >= cin, "pack_dgrad: bad argument");
  const long total = (long)cin_pad * ksize * ksize * k_cout;
  const int grid = (int)((total + 255) / 256 < 148L * 16 ? (total + 255) / 256 : 148L * 16);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (dtype == YB_F16)
    pack_dgrad_weights_kernel<__half><<<grid, 256, 0, st>>>(w_ohwi, cout, cin, ksize, k_cout, cin_pad, (__half*)dst);
  else if (dtype == YB_BF16)
    pack_dgrad_weights_kernel<__nv_bfloat16><<<grid, 256, 0, st>>>(w_ohwi, cout, cin, ksize, k_cout, cin_pad, (__nv_bfloat16*)dst);
  else { set_error("pack_dgrad: bad dtype"); return YB_ERR_UNSUPPORTED; }
  YB_CUDA(cudaGetLastError());
  return YB_OK;
}
