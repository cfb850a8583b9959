// Small layer kernels around the tensor-core conv: the 3-channel stem, weight repack,
// BN folding.  (utils/layer_utils.py:35, utils/misc_utils.py:114-123, model.py:35-41)
#include "common.cuh"

namespace yb {

// ----------------------------------------------------------------------------------
// Stem: darknet53_body/Conv (3 -> 32, 3x3, stride 1, pad 1).  K = 27 is too thin for
// the tensor cores and the layer is HBM-bound (reads 12 B/px, writes 64 B/px), so it
// runs on CUDA cores: a 16x16 pixel tile per CTA, input patch + weights in shared
// memory, 32 fp32 accumulators per thread, fp32 image in -> 16-bit NHWC out.
// ----------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256)
stem_conv_kernel(const float* __restrict__ x, const float* __restrict__ w_ohwi, const float* __restrict__ scale,
                 const float* __restrict__ shift, int H, int W, int leaky, T* __restrict__ out) {
  constexpr int TS = 16, CO = 32;
  __shared__ float s_in[TS + 2][TS + 2][3];
  __shared__ __align__(16) float s_w[27][CO];  // [tap*3+ci][co]
  __shared__ float s_sc[CO], s_sh[CO];
  const int img = blockIdx.z;
  const int ty0 = blockIdx.y * TS, tx0 = blockIdx.x * TS;
  const int tid = threadIdx.x;
  for (int i = tid; i < 27 * CO; i += 256) {
    const int co = i % CO, k = i / CO;       // k = (r*3+s)*3+ci
    s_w[k][co] = w_ohwi[co * 27 + k];
  }
  if (tid < CO) { s_sc[tid] = scale[tid]; s_sh[tid] = shift[tid]; }
  const float* xin = x + (long)img * H * W * 3;
  for (int i = tid; i < (TS + 2) * (TS + 2) * 3; i += 256) {
    const int c = i % 3, px = (i / 3) % (TS + 2), py = i / (3 * (TS + 2));
    const int gy = ty0 + py - 1, gx = tx0 + px - 1;
    float v = 0.f;
    if (gy >= 0 && gy < H && gx >= 0 && gx < W) v = xin[((long)gy * W + gx) * 3 + c];
    s_in[py][px][c] = v;
  }
  __syncthreads();
  const int ly = tid / TS, lx = tid % TS;
  const int oy = ty0 + ly, ox = tx0 + lx;
  if (oy >= H || ox >= W) return;
  float acc[CO];
#pragma unroll
  for (int c = 0; c < CO; ++c) acc[c] = 0.f;
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int s = 0; s < 3; ++s)
#pragma unroll
      for (int ci = 0; ci < 3; ++ci) {
        const float a = s_in[ly + r][lx + s][ci];
        const float4* wr = reinterpret_cast<const float4*>(&s_w[(r * 3 + s) * 3 + ci][0]);
#pragma unroll
        for (int j = 0; j < CO / 4; ++j) {
          const float4 wv = wr[j];
          acc[4 * j + 0] = fmaf(a, wv.x, acc[4 * j + 0]);
          acc[4 * j + 1] = fmaf(a, wv.y, acc[4 * j + 1]);
          acc[4 * j + 2] = fmaf(a, wv.z, acc[4 * j + 2]);
          acc[4 * j + 3] = fmaf(a, wv.w, acc[4 * j + 3]);
        }
      }
  uint4 pk[4];
  uint32_t* pw = reinterpret_cast<uint32_t*>(pk);
#pragma unroll
  for (int j = 0; j < CO / 2; ++j) {
    float a = fmaf(acc[2 * j], s_sc[2 * j], s_sh[2 * j]);
    float b = fmaf(acc[2 * j + 1], s_sc[2 * j + 1], s_sh[2 * j + 1]);
    if (leaky) { a = leaky01(a); b = leaky01(b); }
    pw[j] = Pack2<T>::pack(a, b);
  }
  uint4* op = reinterpret_cast<uint4*>(out + (((long)img * H + oy) * W + ox) * CO);
#pragma unroll
  for (int j = 0; j < 4; ++j) op[j] = pk[j];
}

// ----------------------------------------------------------------------------------
// weight repack: src fp32 in HWIO / OIHW / OHWI  ->  dst OHWI [cout_pad, k, k, cin]
// ----------------------------------------------------------------------------------
template <typename T>
__global__ void pack_weights_kernel(const float* __restrict__ src, int layout, int cout, int cin, int ks,
                                    int cout_pad, T* __restrict__ dst) {
  const long total = (long)cout_pad * ks * ks * cin;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int ci = i % cin;
    const int s = (i / cin) % ks;
    const int r = (i / ((long)cin * ks)) % ks;
    const int co = i / ((long)cin * ks * ks);
    float v = 0.f;
    if (co < cout) {
      long si;
      if (layout == YB_W_HWIO) si = (((long)r * ks + s) * cin + ci) * cout + co;
      else if (layout == YB_W_OIHW) si = (((long)co * cin + ci) * ks + r) * ks + s;
      else si = i;
      v = src[si];
    }
    dst[i] = static_cast<T>(v);
  }
}

__global__ void bn_fold_kernel(const float* gamma, const float* beta, const float* mean, const float* var, int c,
                               float eps, float* scale, float* shift) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < c) {
    const float sc = gamma[i] / sqrtf(var[i] + eps);
    scale[i] = sc;
    shift[i] = beta[i] - mean[i] * sc;
  }
}

// ----------------------------------------------------------------------------------
// fp8 (e4m3) inference: per-output-channel weight quantisation, calibration amax, scale folding
// ----------------------------------------------------------------------------------
// One block per output row co of the packed [cout_pad, k*k*cin] matrix: s_w[co] = amax_co / 448 (1 for an all-zero or
// padding row), q = RN-satfinite e4m3(w / s_w[co]).
__global__ void __launch_bounds__(256) pack_weights_e4m3_kernel(const float* __restrict__ src, int layout, int cout, int cin,
                                                                int ks, uint8_t* __restrict__ dst, float* __restrict__ w_scale) {
  const int co = blockIdx.x;
  const int K = ks * ks * cin;
  auto at = [&](int k) {
    const int ci = k % cin, s = (k / cin) % ks, r = k / (cin * ks);
    long si;
    if (layout == YB_W_HWIO) si = (((long)r * ks + s) * cin + ci) * cout + co;
    else if (layout == YB_W_OIHW) si = (((long)co * cin + ci) * ks + r) * ks + s;
    else si = (long)co * K + k;
    return src[si];
  };
  __shared__ float s_red[8];
  float m = 0.f;
  if (co < cout)
    for (int k = threadIdx.x; k < K; k += blockDim.x) m = fmaxf(m, fabsf(at(k)));
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = m;
  __syncthreads();
  m = s_red[0];
  for (int i = 1; i < 8; ++i) m = fmaxf(m, s_red[i]);
  const float sw = m > 0.f ? m / 448.f : 1.f;
  uint8_t* row = dst + (long)co * K;
  for (int k = threadIdx.x; k < K; k += blockDim.x)
    row[k] = m > 0.f ? (uint8_t)e4m3x2_pack(at(k) / sw, 0.f) : (uint8_t)0;
  if (threadIdx.x == 0) w_scale[co] = sw;
}

// out (zeroed by the caller) = max |x| over a strided [rows, cols] matrix; the max of floats is order-independent, so
// the result is exact and reproducible (the float bits of non-negative values order like unsigned integers)
template <typename T>
__global__ void __launch_bounds__(256) amax_kernel(const T* __restrict__ x, long ld, long rows, int cols,
                                                   unsigned* __restrict__ out) {
  float m = 0.f;
  const long total = rows * cols;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x)
    m = fmaxf(m, fabsf(static_cast<float>(x[(i / cols) * ld + i % cols])));
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0 && m > 0.f) atomicMax(out, __float_as_uint(m));
}

// e4m3 layer: scale = BN scale (1 for the detection heads) x s_in x s_w[c]; BN layers also get shift (the heads' shift
// is their bias and is left alone)
__global__ void fp8_fold_kernel(const float* gamma, const float* beta, const float* mean, const float* var, int c, float eps,
                                float s_in, const float* w_scale, float* scale, float* shift) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= c) return;
  float sc = 1.f;
  if (gamma) {
    sc = gamma[i] / sqrtf(var[i] + eps);
    shift[i] = beta[i] - mean[i] * sc;
  }
  scale[i] = sc * s_in * w_scale[i];
}

int fp8_fold(const float* gamma, const float* beta, const float* mean, const float* var, int c, float eps, float s_in,
             const float* w_scale, float* scale, float* shift, cudaStream_t st) {
  fp8_fold_kernel<<<ceil_div(c, 128), 128, 0, st>>>(gamma, beta, mean, var, c, eps, s_in, w_scale, scale, shift);
  YB_CUDA(cudaGetLastError());
  return YB_OK;
}

}  // namespace yb

using namespace yb;

extern "C" int yb_pack_conv_weights_e4m3(const float* src, int layout, int cout, int cin, int ksize, int cout_pad,
                                         void* dst, float* w_scale, void* stream) {
  YB_REQUIRE(src && dst && w_scale, "pack_e4m3: null pointer");
  YB_REQUIRE(layout >= 0 && layout <= 2, "pack_e4m3: bad layout %d", layout);
  YB_REQUIRE(cout_pad >= cout && cout > 0 && cin > 0 && ksize > 0, "pack_e4m3: bad shape");
  pack_weights_e4m3_kernel<<<cout_pad, 256, 0, static_cast<cudaStream_t>(stream)>>>(src, layout, cout, cin, ksize,
                                                                                    static_cast<uint8_t*>(dst), w_scale);
  YB_CUDA(cudaGetLastError());
  return YB_OK;
}

extern "C" int yb_amax(const void* x, long ld, long rows, int cols, int dtype, float* out, void* stream) {
  YB_REQUIRE(x && out && rows >= 0 && cols > 0 && ld >= cols, "amax: bad argument");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  YB_CUDA(cudaMemsetAsync(out, 0, sizeof(float), st));
  const long total = rows * cols;
  if (total == 0) return YB_OK;
  const long cap = (long)num_sms() * 8;
  const int grid = (int)((total + 255) / 256 < cap ? (total + 255) / 256 : cap);
  unsigned* o = reinterpret_cast<unsigned*>(out);
  if (dtype == YB_F16) amax_kernel<__half><<<grid, 256, 0, st>>>(static_cast<const __half*>(x), ld, rows, cols, o);
  else if (dtype == YB_BF16)
    amax_kernel<__nv_bfloat16><<<grid, 256, 0, st>>>(static_cast<const __nv_bfloat16*>(x), ld, rows, cols, o);
  else if (dtype == YB_F32) amax_kernel<float><<<grid, 256, 0, st>>>(static_cast<const float*>(x), ld, rows, cols, o);
  else { set_error("amax: unsupported dtype %d", dtype); return YB_ERR_UNSUPPORTED; }
  YB_CUDA(cudaGetLastError());
  return YB_OK;
}

extern "C" int yb_stem_conv_fwd(const float* x, const float* w_ohwi, const float* scale, const float* shift, int n,
                                int h, int w, int cout, int dtype, int leaky, void* out, void* stream) {
  YB_REQUIRE(cout == 32, "stem: cout must be 32 (got %d)", cout);
  YB_REQUIRE(x && w_ohwi && scale && shift && out, "stem: null pointer");
  YB_REQUIRE(n > 0 && h > 0 && w > 0 && n <= 65535, "stem: bad shape");
  dim3 grid(ceil_div(w, 16), ceil_div(h, 16), n);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (dtype == YB_F16)
    stem_conv_kernel<__half><<<grid, 256, 0, st>>>(x, w_ohwi, scale, shift, h, w, leaky, static_cast<__half*>(out));
  else if (dtype == YB_BF16)
    stem_conv_kernel<__nv_bfloat16><<<grid, 256, 0, st>>>(x, w_ohwi, scale, shift, h, w, leaky,
                                                        static_cast<__nv_bfloat16*>(out));
  else { set_error("stem: unsupported dtype %d", dtype); return YB_ERR_UNSUPPORTED; }
  YB_CUDA(cudaGetLastError());
  return YB_OK;
}

extern "C" int yb_pack_conv_weights(const float* src, int layout, int cout, int cin, int ksize, int cout_pad,
                                    int dtype, void* dst, void* stream) {
  YB_REQUIRE(src && dst, "pack: null pointer");
  YB_REQUIRE(layout >= 0 && layout <= 2, "pack: bad layout %d", layout);
  YB_REQUIRE(cout_pad >= cout && cout > 0 && cin > 0 && ksize > 0, "pack: bad shape");
  const long total = (long)cout_pad * ksize * ksize * cin;
  const long cap = (long)num_sms() * 16;
  const int grid = (int)((total + 255) / 256 < cap ? (total + 255) / 256 : cap);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (dtype == YB_F16)
    pack_weights_kernel<__half><<<grid, 256, 0, st>>>(src, layout, cout, cin, ksize, cout_pad, static_cast<__half*>(dst));
  else if (dtype == YB_BF16)
    pack_weights_kernel<__nv_bfloat16><<<grid, 256, 0, st>>>(src, layout, cout, cin, ksize, cout_pad,
                                                            static_cast<__nv_bfloat16*>(dst));
  else if (dtype == YB_F32)
    pack_weights_kernel<float><<<grid, 256, 0, st>>>(src, layout, cout, cin, ksize, cout_pad, static_cast<float*>(dst));
  else { set_error("pack: unsupported dtype %d", dtype); return YB_ERR_UNSUPPORTED; }
  YB_CUDA(cudaGetLastError());
  return YB_OK;
}

extern "C" int yb_bn_fold(const float* gamma, const float* beta, const float* mean, const float* var, int c,
                          float eps, float* scale, float* shift, void* stream) {
  YB_REQUIRE(gamma && beta && mean && var && scale && shift && c > 0, "bn_fold: bad argument");
  bn_fold_kernel<<<ceil_div(c, 128), 128, 0, static_cast<cudaStream_t>(stream)>>>(gamma, beta, mean, var, c, eps,
                                                                                  scale, shift);
  YB_CUDA(cudaGetLastError());
  return YB_OK;
}
