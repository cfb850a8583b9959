// Batch-norm (training mode) + leaky-ReLU forward/backward around the tensor-core convs.
// TF semantics (slim.batch_norm fused, model.py:35-41, SURVEY.md B.1): batch mean and
// *biased* variance normalise; moving stats are updated with the *unbiased* variance
// (train.py:108-109 UPDATE_OPS).  The conv epilogue already produced the per-channel
// sum / sum of squares of the raw conv output z (yb_conv2d_fwd stat_sum/stat_sqsum).
//
//   bn_finalize      : sums -> mean/var -> scale/shift (+ saved mean/invstd, moving update)
//   bn_act_apply     : a = leaky(z*scale+shift) (+ residual), optional 2x-upsample store
//   bn_bwd_reduce    : dbeta = sum(dact), dgamma = sum(dact * zhat), dact = dA * leaky'(y)
//   bn_bwd_apply     : dz = gamma*invstd*(dact - dbeta/M - zhat*dgamma/M), optional
//                      zero-insertion (dilated) store for the dgrad of stride-2 convs
// M is the number of rows the statistics cover: n*h*w on one device, replicas*n*h*w under synchronised BN, where
// the sums are all-reduced across equal-shaped ranks between the producing and the consuming kernel.
//   col_sum          : bias gradient of the detection convs
// All are HBM-bound streaming kernels over [rows, C] NHWC 16-bit tensors (C % 8 == 0):
// a thread owns 8 consecutive channels (one 16-byte load), a block a slab of rows.
#include "common.cuh"
#include <initializer_list>

namespace yb {

// Batch statistics -> (mean, biased var, invstd, scale, shift) and the moving-statistics update.  Shared by the
// finalize kernel and the fused statistics + apply kernel, which must agree bit for bit: every product and sum is
// rounded explicitly, so no FMA contraction the compiler may pick differently in the two contexts changes a result.
__device__ __forceinline__ void bn_batch_coeffs(float su, float sq, float count, float ga, float be, float eps, float& mean,
                                                float& var, float& invstd, float& sc, float& sh) {
  mean = __fdiv_rn(su, count);
  var = fmaxf(__fsub_rn(__fdiv_rn(sq, count), __fmul_rn(mean, mean)), 0.f);   // biased
  invstd = rsqrtf(__fadd_rn(var, eps));
  sc = __fmul_rn(ga, invstd);
  sh = __fsub_rn(be, __fmul_rn(mean, sc));
}
__device__ __forceinline__ void bn_moving_update(float& mm, float& mv, float mean, float var, float count, float decay) {
  const float unb = count > 1.f ? __fdiv_rn(__fmul_rn(var, count), __fsub_rn(count, 1.f)) : var;   // unbiased
  const float keep = __fsub_rn(1.f, decay);
  mm = __fadd_rn(__fmul_rn(mm, decay), __fmul_rn(keep, mean));
  mv = __fadd_rn(__fmul_rn(mv, decay), __fmul_rn(keep, unb));
}

__global__ void bn_finalize_kernel(const float* __restrict__ sum, const float* __restrict__ sqsum, float count, int c,
                                   const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                                   float decay, float* moving_mean, float* moving_var, float* scale, float* shift,
                                   float* save_mean, float* save_invstd) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= c) return;
  if (sum == nullptr) {
    // frozen BN (forward(is_training=False) under a gradient tape): normalise with the MOVING statistics, which are
    // constants of the backward pass and are not updated
    const float invstd = rsqrtf(moving_var[i] + eps);
    const float sc = gamma[i] * invstd;
    scale[i] = sc;
    shift[i] = beta[i] - moving_mean[i] * sc;
    save_mean[i] = moving_mean[i];
    save_invstd[i] = invstd;
    return;
  }
  float mean, var, invstd, sc, sh;
  bn_batch_coeffs(sum[i], sqsum[i], count, gamma[i], beta[i], eps, mean, var, invstd, sc, sh);
  scale[i] = sc;
  shift[i] = sh;
  save_mean[i] = mean;
  save_invstd[i] = invstd;
  if (moving_mean) bn_moving_update(moving_mean[i], moving_var[i], mean, var, count, decay);
}

struct RowGeom {
  long rows;        // n*h*w
  int h, w;         // spatial (for the upsample / dilate address maps)
  int c;
};
struct StreamGeom {
  int cv;             // channel vectors per row (c / CPT)
  int lanes;          // row lanes per block (256 / cv)
  long rows_per_block;
};

// CPT consecutive 16-bit channels of one row: one 16-byte (CPT = 8) or 8-byte (CPT = 4) access
template <typename T, int CPT> struct ChanVec;
template <typename T> struct ChanVec<T, 8> {
  using V = uint4;
  static __device__ __forceinline__ void unpack(const V& u, float (&v)[8]) {
    float2 f;
    f = Pack2<T>::unpack(u.x); v[0] = f.x; v[1] = f.y;
    f = Pack2<T>::unpack(u.y); v[2] = f.x; v[3] = f.y;
    f = Pack2<T>::unpack(u.z); v[4] = f.x; v[5] = f.y;
    f = Pack2<T>::unpack(u.w); v[6] = f.x; v[7] = f.y;
  }
  static __device__ __forceinline__ V pack(const float (&v)[8]) {
    V u;
    u.x = Pack2<T>::pack(v[0], v[1]); u.y = Pack2<T>::pack(v[2], v[3]);
    u.z = Pack2<T>::pack(v[4], v[5]); u.w = Pack2<T>::pack(v[6], v[7]);
    return u;
  }
};
template <typename T> struct ChanVec<T, 4> {
  using V = uint2;
  static __device__ __forceinline__ void unpack(const V& u, float (&v)[4]) {
    float2 f;
    f = Pack2<T>::unpack(u.x); v[0] = f.x; v[1] = f.y;
    f = Pack2<T>::unpack(u.y); v[2] = f.x; v[3] = f.y;
  }
  static __device__ __forceinline__ V pack(const float (&v)[4]) {
    V u;
    u.x = Pack2<T>::pack(v[0], v[1]); u.y = Pack2<T>::pack(v[2], v[3]);
    return u;
  }
};
template <typename T, int CPT>
__device__ __forceinline__ typename ChanVec<T, CPT>::V ldv(const T* p) {
  return *reinterpret_cast<const typename ChanVec<T, CPT>::V*>(p);
}
template <typename T, int CPT>
__device__ __forceinline__ void stv(T* p, const float (&v)[CPT]) {
  *reinterpret_cast<typename ChanVec<T, CPT>::V*>(p) = ChanVec<T, CPT>::pack(v);
}
// row index in the 2x-upsampled [n, 2h, 2w] grid of the top-left copy of row r of [n, h, w]
__device__ __forceinline__ long up_row(long r, int h, int w) {
  const long q = r % w, pp = (r / w) % h, img = r / ((long)w * h);
  return ((img * 2 * h + 2 * pp) * (2L * w)) + 2 * q;
}

// ---- streaming kernels: thread = (CPT-channel vector, row lane); per-channel coefficients live in registers, rows are
// ---- walked R at a time so several vector loads are in flight per thread.
// Launch shape: ONE balanced wave of (SM count) x BPS co-resident blocks.  The first version
// launched 4 blocks per SM with 3 resident (a 1/3-occupancy tail wave on the large layers: 0.6 of the HBM peak), spilled
// (85-register cap against 40 coefficient registers) and fetched the per-channel coefficients with 56 scalar loads per
// thread whose 32-byte stride makes every warp instruction touch 32 sectors — on the 13x13 / 26x26 layers, where a
// thread only streams 8-16 rows, that prologue cost as much as the data (15 us floor per launch, 72 x 2 launches a step).
// Two shapes are built: CPT 8 / R 4 / 2 blocks per SM (16-byte accesses, ~120 registers; the default) and CPT 4 / R 8 /
// 3 blocks per SM (8-byte accesses, half the coefficient registers, 1.5x the bytes in flight per SM; YB_BN_CPT=4).

// CPT consecutive per-channel fp32 coefficients (c0 % CPT == 0): 16-byte loads when every array is 16-byte aligned
template <int CPT>
__device__ __forceinline__ void ldc(const float* __restrict__ p, int vec, float (&v)[CPT]) {
  if (vec) {
#pragma unroll
    for (int q = 0; q < CPT / 4; ++q) {
      const float4 a = __ldg(reinterpret_cast<const float4*>(p) + q);
      v[4 * q] = a.x; v[4 * q + 1] = a.y; v[4 * q + 2] = a.z; v[4 * q + 3] = a.w;
    }
  } else {
#pragma unroll
    for (int j = 0; j < CPT; ++j) v[j] = __ldg(p + j);
  }
}
template <int CPT>
__device__ __forceinline__ void stc(float* __restrict__ p, int vec, const float (&v)[CPT]) {
  if (vec) {
#pragma unroll
    for (int q = 0; q < CPT / 4; ++q)
      reinterpret_cast<float4*>(p)[q] = make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]);
  } else {
#pragma unroll
    for (int j = 0; j < CPT; ++j) p[j] = v[j];
  }
}
// gradient of a row the forward stored 2x-upsampled: the fp32 sum of its 4 copies
template <typename T, int CPT>
__device__ __forceinline__ void load_dA_up(const T* dA, long dA_ld, long r, int c0, const RowGeom& g, float (&v)[CPT]) {
  const long b = up_row(r, g.h, g.w);
  const long W2 = 2L * g.w;
  float t0[CPT], t1[CPT], t2[CPT];
  ChanVec<T, CPT>::unpack(ldv<T, CPT>(dA + b * dA_ld + c0), v);
  ChanVec<T, CPT>::unpack(ldv<T, CPT>(dA + (b + 1) * dA_ld + c0), t0);
  ChanVec<T, CPT>::unpack(ldv<T, CPT>(dA + (b + W2) * dA_ld + c0), t1);
  ChanVec<T, CPT>::unpack(ldv<T, CPT>(dA + (b + W2 + 1) * dA_ld + c0), t2);
#pragma unroll
  for (int j = 0; j < CPT; ++j) v[j] += t0[j] + t1[j] + t2[j];
}

// Batch statistics -> scale/shift folded into the apply kernel (FIN): every thread derives the coefficients of its
// channels from the conv epilogue's sums (same arithmetic as bn_finalize_kernel, so the two paths are bit-identical);
// the row-lane-0 threads of block 0 also store scale/shift/mean/invstd for the backward and update the moving statistics.
// 72 six-microsecond bn_finalize launches per training step disappear.
struct BnFin {
  const float* sum; const float* sqsum;     // NULL: frozen BN (moving statistics)
  const float* gamma; const float* beta;
  float* moving_mean; float* moving_var;
  float* scale; float* shift; float* save_mean; float* save_invstd;
  float count, eps, decay;
};

template <typename T, int CPT, int R, int BPS, bool FIN>
__global__ void __launch_bounds__(256, BPS)
bn_act_apply_kernel(const T* __restrict__ z, long z_ld, const float* __restrict__ scale, const float* __restrict__ shift,
                    const T* __restrict__ res, long res_ld, T* __restrict__ out, long out_ld, RowGeom g, StreamGeom sg,
                    int leaky, int upsample, int vec, BnFin f) {
  using CV = ChanVec<T, CPT>;
  const int cvi = threadIdx.x % sg.cv, lane_r = threadIdx.x / sg.cv;
  const int c0 = cvi * CPT;
  float sc[CPT], sh[CPT];
  if (FIN) {
    float ga[CPT], be[CPT], mean[CPT], invstd[CPT], var[CPT];
    ldc<CPT>(f.gamma + c0, vec, ga); ldc<CPT>(f.beta + c0, vec, be);
    if (f.sum == nullptr) {
      ldc<CPT>(f.moving_mean + c0, vec, mean); ldc<CPT>(f.moving_var + c0, vec, var);
#pragma unroll
      for (int j = 0; j < CPT; ++j) invstd[j] = rsqrtf(var[j] + f.eps);
    } else {
      float su[CPT], sq[CPT];
      ldc<CPT>(f.sum + c0, vec, su); ldc<CPT>(f.sqsum + c0, vec, sq);
#pragma unroll
      for (int j = 0; j < CPT; ++j) bn_batch_coeffs(su[j], sq[j], f.count, ga[j], be[j], f.eps, mean[j], var[j], invstd[j], sc[j], sh[j]);
    }
    if (f.sum == nullptr) {
#pragma unroll
      for (int j = 0; j < CPT; ++j) { sc[j] = ga[j] * invstd[j]; sh[j] = be[j] - mean[j] * sc[j]; }
    }
    if (blockIdx.x == 0 && lane_r == 0) {
      stc<CPT>(f.scale + c0, vec, sc); stc<CPT>(f.shift + c0, vec, sh);
      stc<CPT>(f.save_mean + c0, vec, mean); stc<CPT>(f.save_invstd + c0, vec, invstd);
      if (f.sum != nullptr && f.moving_mean != nullptr) {
        float mm[CPT], mv[CPT];
        ldc<CPT>(f.moving_mean + c0, vec, mm); ldc<CPT>(f.moving_var + c0, vec, mv);
#pragma unroll
        for (int j = 0; j < CPT; ++j) bn_moving_update(mm[j], mv[j], mean[j], var[j], f.count, f.decay);
        stc<CPT>(f.moving_mean + c0, vec, mm); stc<CPT>(f.moving_var + c0, vec, mv);
      }
    }
  } else {
    ldc<CPT>(scale + c0, vec, sc); ldc<CPT>(shift + c0, vec, sh);
  }
  const long r0 = blockIdx.x * sg.rows_per_block, r1 = min(r0 + sg.rows_per_block, g.rows);
  for (long rb = r0 + lane_r; rb < r1; rb += (long)R * sg.lanes) {
    typename CV::V zq[R], rq[R];
#pragma unroll
    for (int u = 0; u < R; ++u) {
      const long r = rb + (long)u * sg.lanes;
      if (r < r1) {
        zq[u] = ldv<T, CPT>(z + r * z_ld + c0);
        if (res) rq[u] = ldv<T, CPT>(res + r * res_ld + c0);
      }
    }
#pragma unroll
    for (int u = 0; u < R; ++u) {
      const long r = rb + (long)u * sg.lanes;
      if (r >= r1) break;
      float v[CPT], rv[CPT];
      CV::unpack(zq[u], v);
      if (res) CV::unpack(rq[u], rv);
#pragma unroll
      for (int j = 0; j < CPT; ++j) {
        float y = fmaf(v[j], sc[j], sh[j]);
        if (leaky) y = leaky01(y);
        if (res) y += rv[j];
        v[j] = y;
      }
      if (!upsample) {
        stv<T, CPT>(out + r * out_ld + c0, v);
      } else {
        const long bb = up_row(r, g.h, g.w);
        const long W2 = 2L * g.w;
        stv<T, CPT>(out + bb * out_ld + c0, v); stv<T, CPT>(out + (bb + 1) * out_ld + c0, v);
        stv<T, CPT>(out + (bb + W2) * out_ld + c0, v); stv<T, CPT>(out + (bb + W2 + 1) * out_ld + c0, v);
      }
    }
  }
}

// Stage 1: every block reduces its row slab to per-channel partial sums.  With a (zero-initialised) workspace the
// partials are added into one of BN_SLOTS rows [slot][2][c] and the LAST block to finish (ticket counter) sums the
// rows, writes dgamma/dbeta and zeroes the rows again; without one they are added atomically to dgamma/dbeta
// (grid-deep same-address atomics: slow, kept for callers without a workspace).
static constexpr int BN_SLOTS = 16;

template <typename T, int CPT, int R, int BPS>
__global__ void __launch_bounds__(256, BPS)
bn_bwd_reduce_kernel(const T* __restrict__ dA, long dA_ld, const T* __restrict__ z, long z_ld,
                     const float* __restrict__ scale, const float* __restrict__ shift,
                     const float* __restrict__ save_mean, const float* __restrict__ save_invstd, RowGeom g,
                     StreamGeom sg, int leaky, int upsample, int vec, float* __restrict__ dgamma,
                     float* __restrict__ dbeta, float* __restrict__ partial, unsigned int* __restrict__ ticket,
                     float* __restrict__ xg, float* __restrict__ xb) {
  using CV = ChanVec<T, CPT>;
  __shared__ float s_g[256][CPT + 1], s_b[256][CPT + 1];
  __shared__ unsigned int s_last;
  const int cvi = threadIdx.x % sg.cv, lane_r = threadIdx.x / sg.cv;
  const int c0 = cvi * CPT;
  // per-channel coefficients live in registers (the first version re-loaded four of them per ELEMENT through the LSU,
  // which made this kernel 2x slower than bn_bwd_apply on the same data).  The invstd factor of
  // zhat = (z - mean) * invstd is folded in once per block at the end.
  float sc[CPT], sh[CPT];
  ldc<CPT>(scale + c0, vec, sc); ldc<CPT>(shift + c0, vec, sh);
  float ag[CPT], ab[CPT];
#pragma unroll
  for (int j = 0; j < CPT; ++j) ag[j] = ab[j] = 0.f;
  const long r0 = blockIdx.x * sg.rows_per_block, r1 = min(r0 + sg.rows_per_block, g.rows);
  for (long rb = r0 + lane_r; rb < r1; rb += (long)R * sg.lanes) {
    typename CV::V zq[R], dq[R];
#pragma unroll
    for (int u = 0; u < R; ++u) {
      const long r = rb + (long)u * sg.lanes;
      if (r < r1) { zq[u] = ldv<T, CPT>(z + r * z_ld + c0); if (!upsample) dq[u] = ldv<T, CPT>(dA + r * dA_ld + c0); }
    }
#pragma unroll
    for (int u = 0; u < R; ++u) {
      if (rb + (long)u * sg.lanes >= r1) break;
      float zv[CPT], dv[CPT];
      CV::unpack(zq[u], zv);
      if (!upsample) CV::unpack(dq[u], dv);
      else load_dA_up<T, CPT>(dA, dA_ld, rb + (long)u * sg.lanes, c0, g, dv);
#pragma unroll
      for (int j = 0; j < CPT; ++j) {
        const float y = fmaf(zv[j], sc[j], sh[j]);
        const float da = (leaky && y <= 0.f) ? 0.1f * dv[j] : dv[j];
        ab[j] += da;
        ag[j] = fmaf(da, zv[j], ag[j]);        // sum(da * z); centred and scaled below
      }
    }
  }
  {
    float mu[CPT], is[CPT];
    ldc<CPT>(save_mean + c0, vec, mu); ldc<CPT>(save_invstd + c0, vec, is);
#pragma unroll
    for (int j = 0; j < CPT; ++j)   // sum(da * zhat) = invstd * (sum(da * z) - mean * sum(da))   (linear: exact per block)
      ag[j] = (ag[j] - mu[j] * ab[j]) * is[j];
  }
#pragma unroll
  for (int j = 0; j < CPT; ++j) { s_g[threadIdx.x][j] = ag[j]; s_b[threadIdx.x][j] = ab[j]; }
  __syncthreads();
  if (lane_r == 0) {
    for (int y = 1; y < sg.lanes; ++y) {
#pragma unroll
      for (int j = 0; j < CPT; ++j) { ag[j] += s_g[y * sg.cv + cvi][j]; ab[j] += s_b[y * sg.cv + cvi][j]; }
    }
    if (partial == nullptr) {
#pragma unroll
      for (int j = 0; j < CPT; ++j) { atomicAdd(dgamma + c0 + j, ag[j]); atomicAdd(dbeta + c0 + j, ab[j]); }
    } else {
      // BN_SLOTS partial rows (zero on entry): ~grid/BN_SLOTS-deep atomics per address instead of grid-deep, and the
      // final pass reads BN_SLOTS x 2c floats instead of grid x 2c (which made one SM stream megabytes: r01_i)
      float* pg = partial + (long)(blockIdx.x % BN_SLOTS) * 2 * g.c;
#pragma unroll
      for (int j = 0; j < CPT; ++j) { atomicAdd(pg + c0 + j, ag[j]); atomicAdd(pg + g.c + c0 + j, ab[j]); }
    }
  }
  if (partial == nullptr) return;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) s_last = (atomicAdd(ticket, 1u) == gridDim.x - 1) ? 1u : 0u;
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  for (int c = threadIdx.x; c < 2 * g.c; c += 256) {
    float v[BN_SLOTS];
#pragma unroll
    for (int sl = 0; sl < BN_SLOTS; ++sl) v[sl] = __ldcg(partial + (long)sl * 2 * g.c + c);
    float acc = 0.f;
#pragma unroll
    for (int sl = 0; sl < BN_SLOTS; ++sl) { acc += v[sl]; partial[(long)sl * 2 * g.c + c] = 0.f; }   // re-armed
    if (c < g.c) { dgamma[c] = acc; if (xg) xg[c] = acc; }
    else { dbeta[c - g.c] = acc; if (xb) xb[c - g.c] = acc; }
  }
  if (threadIdx.x == 0) *ticket = 0u;   // ready for the next launch
}

template <typename T, int CPT, int R, int BPS>
__global__ void __launch_bounds__(256, BPS)
bn_bwd_apply_kernel(const T* __restrict__ dA, long dA_ld, const T* __restrict__ z, long z_ld,
                    const float* __restrict__ gamma, const float* __restrict__ scale, const float* __restrict__ shift,
                    const float* __restrict__ save_mean, const float* __restrict__ save_invstd,
                    const float* __restrict__ dgamma, const float* __restrict__ dbeta, RowGeom g, StreamGeom sg,
                    int leaky, int upsample, int dilate, int vec, float count, T* __restrict__ dz, long dz_ld) {
  using CV = ChanVec<T, CPT>;
  const int cvi = threadIdx.x % sg.cv, lane_r = threadIdx.x / sg.cv;
  const int c0 = cvi * CPT;
  const float inv_m = 1.f / count;
  // dz = k1*dact + k2*z + k3   with   k1 = gamma*invstd, k2 = -k1*invstd*dgamma/M, k3 = -k1*dbeta/M - k2*mean
  float sc[CPT], sh[CPT], k1[CPT], k2[CPT], k3[CPT];
  ldc<CPT>(scale + c0, vec, sc); ldc<CPT>(shift + c0, vec, sh);
  {
    float is[CPT], ga[CPT], dg[CPT], db[CPT], mu[CPT];
    ldc<CPT>(save_invstd + c0, vec, is); ldc<CPT>(gamma + c0, vec, ga); ldc<CPT>(dgamma + c0, vec, dg);
    ldc<CPT>(dbeta + c0, vec, db); ldc<CPT>(save_mean + c0, vec, mu);
#pragma unroll
    for (int j = 0; j < CPT; ++j) {
      k1[j] = ga[j] * is[j];
      k2[j] = -k1[j] * is[j] * dg[j] * inv_m;
      k3[j] = -k1[j] * db[j] * inv_m - k2[j] * mu[j];
    }
  }
  const long r0 = blockIdx.x * sg.rows_per_block, r1 = min(r0 + sg.rows_per_block, g.rows);
  for (long rb = r0 + lane_r; rb < r1; rb += (long)R * sg.lanes) {
    typename CV::V zq[R], dq[R];
#pragma unroll
    for (int u = 0; u < R; ++u) {
      const long r = rb + (long)u * sg.lanes;
      if (r < r1) { zq[u] = ldv<T, CPT>(z + r * z_ld + c0); if (!upsample) dq[u] = ldv<T, CPT>(dA + r * dA_ld + c0); }
    }
#pragma unroll
    for (int u = 0; u < R; ++u) {
      const long r = rb + (long)u * sg.lanes;
      if (r >= r1) break;
      float zv[CPT], dv[CPT], o[CPT];
      CV::unpack(zq[u], zv);
      if (!upsample) CV::unpack(dq[u], dv);
      else load_dA_up<T, CPT>(dA, dA_ld, r, c0, g, dv);
#pragma unroll
      for (int j = 0; j < CPT; ++j) {
        const float y = fmaf(zv[j], sc[j], sh[j]);
        const float da = (leaky && y <= 0.f) ? 0.1f * dv[j] : dv[j];
        o[j] = fmaf(k1[j], da, fmaf(k2[j], zv[j], k3[j]));
      }
      const long orow = dilate ? up_row(r, g.h, g.w) : r;   // (2p, 2q) of a zero-initialised [n,2h,2w] buffer
      stv<T, CPT>(dz + orow * dz_ld + c0, o);
    }
  }
}

// kernel shape: 8 channels per thread (16-byte accesses) unless YB_BN_CPT=4, whose 8-byte accesses double the
// load/store instructions per byte.
static int bn_cpt(int c) {
  const char* o = opt("YB_BN_CPT");
  if (c > 1024 || c < 32) return 8;
  return (o && o[0] == '4') ? 4 : 8;
}
// the launch shape yb_bn_schedule reports for this device (the callers have validated rows and c)
static StreamGeom stream_geom(long rows, int c, int* cpt, int* grid) {
  yb_bn_schedule_info s;
  yb_bn_schedule(rows, c, num_sms(), &s);
  StreamGeom sg;
  sg.cv = s.cv;
  sg.lanes = s.lanes;
  sg.rows_per_block = s.rows_per_block;
  *cpt = s.cpt;
  *grid = s.grid;
  return sg;
}
static int aligned16(std::initializer_list<const void*> ps) {
  for (const void* q : ps) if (q && (reinterpret_cast<uintptr_t>(q) & 15)) return 0;
  return 1;
}

template <typename T>
__global__ void __launch_bounds__(256)
col_sum_kernel(const T* __restrict__ x, long ld, long rows, int c, long rows_per_block, float* __restrict__ out,
               float* __restrict__ out_sq) {
  // block (32, 8): 32 channels x 8 row lanes
  __shared__ float s[8][33], s2[8][33];
  const int ch = blockIdx.y * 32 + threadIdx.x;
  float a = 0.f, a2 = 0.f;
  const long r0 = blockIdx.x * rows_per_block, r1 = min(r0 + rows_per_block, rows);
  if (ch < c)
    for (long r = r0 + threadIdx.y; r < r1; r += 8) {
      const float v = static_cast<float>(x[r * ld + ch]);
      a += v; a2 += v * v;
    }
  s[threadIdx.y][threadIdx.x] = a; s2[threadIdx.y][threadIdx.x] = a2;
  __syncthreads();
  if (threadIdx.y == 0 && ch < c) {
    for (int y = 1; y < 8; ++y) { a += s[y][threadIdx.x]; a2 += s2[y][threadIdx.x]; }
    atomicAdd(out + ch, a);
    if (out_sq) atomicAdd(out_sq + ch, a2);
  }
}

}  // namespace yb

using namespace yb;

#define YB_BN_COMMON_CHECK(name)                                                                         \
  YB_REQUIRE(n > 0 && h > 0 && w > 0 && c >= 8 && c <= 2048 && (c & (c - 1)) == 0, name ": channels must be a power of two in [8, 2048]"); \
  YB_REQUIRE(dtype == YB_F16 || dtype == YB_BF16, name ": dtype must be f16 or bf16");

// one balanced wave: at most (SM count) x bps co-resident blocks, every row lane of a block gets >= 1 row
extern "C" int yb_bn_schedule(long rows, int c, int sm_count, yb_bn_schedule_info* info) {
  YB_REQUIRE(info && sm_count > 0 && rows > 0, "bn_schedule: bad argument");
  YB_REQUIRE(c >= 8 && c <= 2048 && (c & (c - 1)) == 0, "bn_schedule: channels must be a power of two in [8, 2048]");
  const int cpt = bn_cpt(c);
  info->cpt = cpt;
  info->r = cpt == 4 ? 8 : 4;                 // the YB_BN_SHAPES instantiations below
  info->blocks_per_sm = cpt == 4 ? 3 : 2;
  info->cv = c / cpt;
  info->lanes = 256 / info->cv;
  if (info->lanes < 1) info->lanes = 1;
  const long blocks = (long)sm_count * info->blocks_per_sm;
  long rpb = (rows + blocks - 1) / blocks;
  rpb = (rpb + info->lanes - 1) / info->lanes * info->lanes;
  info->rows_per_block = rpb;
  info->grid = (int)((rows + rpb - 1) / rpb);
  return YB_OK;
}

extern "C" int yb_bn_finalize(const float* sum, const float* sqsum, long count, int c, const float* gamma,
                              const float* beta, float eps, float decay, float* moving_mean, float* moving_var,
                              float* scale, float* shift, float* save_mean, float* save_invstd, void* stream) {
  YB_REQUIRE(gamma && beta && scale && shift && save_mean && save_invstd && c > 0 && count > 0, "bn_finalize: bad argument");
  YB_REQUIRE((sum == nullptr) == (sqsum == nullptr), "bn_finalize: sum/sqsum must both be given (both NULL: frozen BN)");
  YB_REQUIRE((moving_mean == nullptr) == (moving_var == nullptr), "bn_finalize: moving_mean/var must both be given");
  YB_REQUIRE(sum || moving_mean, "bn_finalize: frozen BN needs the moving statistics");
  bn_finalize_kernel<<<ceil_div(c, 128), 128, 0, static_cast<cudaStream_t>(stream)>>>(
      sum, sqsum, (float)count, c, gamma, beta, eps, decay, moving_mean, moving_var, scale, shift, save_mean, save_invstd);
  YB_CUDA(cudaGetLastError());
  return YB_OK;
}

// shape dispatch: (CPT 4, R 8, 3 blocks / SM) or (CPT 8, R 4, 2 blocks / SM)
#define YB_BN_SHAPES(T, LAUNCH)            \
  if (cpt == 4) { LAUNCH(T, 4, 8, 3); }    \
  else { LAUNCH(T, 8, 4, 2); }
#define YB_BN_DTYPES(LAUNCH)                                   \
  if (dtype == YB_F16) { YB_BN_SHAPES(__half, LAUNCH) }        \
  else { YB_BN_SHAPES(__nv_bfloat16, LAUNCH) }

static int launch_act_apply(const void* z, long z_ld, const float* scale, const float* shift, const void* res,
                            long res_ld, void* out, long out_ld, int n, int h, int w, int c, int dtype, int leaky,
                            int upsample2x, const BnFin* fin, cudaStream_t st) {
  RowGeom g{(long)n * h * w, h, w, c};
  int grid, cpt;
  const StreamGeom sg = stream_geom(g.rows, c, &cpt, &grid);
  BnFin f; memset(&f, 0, sizeof(f));
  int vec = aligned16({scale, shift});
  if (fin) {
    f = *fin;
    vec = aligned16({f.sum, f.sqsum, f.gamma, f.beta, f.moving_mean, f.moving_var, f.scale, f.shift, f.save_mean, f.save_invstd});
  }
#define YB_ACT_LAUNCH(T, CPT, R, BPS)                                                                                   \
  if (fin) bn_act_apply_kernel<T, CPT, R, BPS, true><<<grid, 256, 0, st>>>((const T*)z, z_ld, scale, shift, (const T*)res, \
                                                          res_ld, (T*)out, out_ld, g, sg, leaky, upsample2x, vec, f);   \
  else bn_act_apply_kernel<T, CPT, R, BPS, false><<<grid, 256, 0, st>>>((const T*)z, z_ld, scale, shift, (const T*)res,  \
                                                          res_ld, (T*)out, out_ld, g, sg, leaky, upsample2x, vec, f)
  YB_BN_DTYPES(YB_ACT_LAUNCH)
#undef YB_ACT_LAUNCH
  YB_CUDA(cudaGetLastError());
  return YB_OK;
}

extern "C" int yb_bn_act_apply(const void* z, long z_ld, const float* scale, const float* shift, const void* res,
                               long res_ld, void* out, long out_ld, int n, int h, int w, int c, int dtype, int leaky,
                               int upsample2x, void* stream) {
  YB_BN_COMMON_CHECK("bn_act_apply");
  YB_REQUIRE(z && scale && shift && out, "bn_act_apply: null pointer");
  return launch_act_apply(z, z_ld, scale, shift, res, res_ld, out, out_ld, n, h, w, c, dtype, leaky, upsample2x, nullptr,
                          static_cast<cudaStream_t>(stream));
}

// yb_bn_finalize + yb_bn_act_apply in one launch (same arguments, same results): the training forward of a BN conv
namespace yb {
// count: the rows the sums cover (n*h*w, or replicas*n*h*w when the sums were all-reduced across ranks)
int bn_stats_act_apply_n(const void* z, long z_ld, const float* sum, const float* sqsum, long count, const float* gamma,
                         const float* beta, float eps, float decay, float* moving_mean, float* moving_var, float* scale,
                         float* shift, float* save_mean, float* save_invstd, const void* res, long res_ld, void* out,
                         long out_ld, int n, int h, int w, int c, int dtype, int leaky, int upsample2x, void* stream) {
  YB_BN_COMMON_CHECK("bn_stats_act_apply");
  YB_REQUIRE(count >= (long)n * h * w, "bn_stats_act_apply: count must cover the local rows");
  YB_REQUIRE(z && out && gamma && beta && scale && shift && save_mean && save_invstd, "bn_stats_act_apply: null pointer");
  YB_REQUIRE((sum == nullptr) == (sqsum == nullptr), "bn_stats_act_apply: sum/sqsum must both be given (both NULL: frozen BN)");
  YB_REQUIRE((moving_mean == nullptr) == (moving_var == nullptr), "bn_stats_act_apply: moving_mean/var must both be given");
  YB_REQUIRE(sum || moving_mean, "bn_stats_act_apply: frozen BN needs the moving statistics");
  BnFin f{sum, sqsum, gamma, beta, moving_mean, moving_var, scale, shift, save_mean, save_invstd, (float)count, eps, decay};
  return launch_act_apply(z, z_ld, nullptr, nullptr, res, res_ld, out, out_ld, n, h, w, c, dtype, leaky, upsample2x, &f,
                          static_cast<cudaStream_t>(stream));
}
}  // namespace yb

extern "C" int yb_bn_stats_act_apply(const void* z, long z_ld, const float* sum, const float* sqsum, const float* gamma,
                                     const float* beta, float eps, float decay, float* moving_mean, float* moving_var,
                                     float* scale, float* shift, float* save_mean, float* save_invstd, const void* res,
                                     long res_ld, void* out, long out_ld, int n, int h, int w, int c, int dtype,
                                     int leaky, int upsample2x, void* stream) {
  return bn_stats_act_apply_n(z, z_ld, sum, sqsum, (long)n * h * w, gamma, beta, eps, decay, moving_mean, moving_var,
                              scale, shift, save_mean, save_invstd, res, res_ld, out, out_ld, n, h, w, c, dtype, leaky,
                              upsample2x, stream);
}

extern "C" int yb_bn_bwd_reduce_workspace_bytes(size_t* bytes) {
  YB_REQUIRE(bytes, "bn_bwd_reduce_workspace_bytes: null pointer");
  *bytes = 256 + (size_t)16 * 2 * 2048 * sizeof(float);   // ticket + BN_SLOTS x [2][c <= 2048]
  return YB_OK;
}

namespace yb {
// xg / xb (optional, both or neither, needs a workspace): the final block also stores the two sums there — the
// exchange slab a synchronised-BN caller all-reduces while dgamma / dbeta keep the local sums
int bn_bwd_reduce_x(const void* dA, long dA_ld, const void* z, long z_ld, const float* scale, const float* shift,
                    const float* save_mean, const float* save_invstd, int n, int h, int w, int c, int dtype, int leaky,
                    int upsample2x, float* dgamma, float* dbeta, void* workspace, float* xg, float* xb, void* stream) {
  YB_BN_COMMON_CHECK("bn_bwd_reduce");
  YB_REQUIRE(dA && z && scale && shift && save_mean && save_invstd && dgamma && dbeta, "bn_bwd_reduce: null pointer");
  YB_REQUIRE((xg == nullptr) == (xb == nullptr) && (xg == nullptr || workspace), "bn_bwd_reduce: bad exchange slab");
  RowGeom g{(long)n * h * w, h, w, c};
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int grid, cpt;
  const StreamGeom sg = stream_geom(g.rows, c, &cpt, &grid);
  // workspace (zero-initialised once by the caller): [0,256) ticket counter, then per-block partials
  unsigned int* ticket = static_cast<unsigned int*>(workspace);
  float* partial = workspace ? reinterpret_cast<float*>(static_cast<uint8_t*>(workspace) + 256) : nullptr;
  if (!workspace) {
    YB_CUDA(cudaMemsetAsync(dgamma, 0, c * 4, st));
    YB_CUDA(cudaMemsetAsync(dbeta, 0, c * 4, st));
  }
  const int vec = aligned16({scale, shift, save_mean, save_invstd});
#define YB_RED_LAUNCH(T, CPT, R, BPS)                                                                                  \
  bn_bwd_reduce_kernel<T, CPT, R, BPS><<<grid, 256, 0, st>>>((const T*)dA, dA_ld, (const T*)z, z_ld, scale, shift,      \
                                                             save_mean, save_invstd, g, sg, leaky, upsample2x, vec,   \
                                                             dgamma, dbeta, partial, ticket, xg, xb)
  YB_BN_DTYPES(YB_RED_LAUNCH)
#undef YB_RED_LAUNCH
  YB_CUDA(cudaGetLastError());
  return YB_OK;
}
}  // namespace yb

extern "C" int yb_bn_bwd_reduce(const void* dA, long dA_ld, const void* z, long z_ld, const float* scale,
                                const float* shift, const float* save_mean, const float* save_invstd, int n, int h,
                                int w, int c, int dtype, int leaky, int upsample2x, float* dgamma, float* dbeta,
                                void* workspace, void* stream) {
  return bn_bwd_reduce_x(dA, dA_ld, z, z_ld, scale, shift, save_mean, save_invstd, n, h, w, c, dtype, leaky, upsample2x,
                         dgamma, dbeta, workspace, nullptr, nullptr, stream);
}

namespace yb {
// count: the rows dgamma / dbeta cover (n*h*w, or replicas*n*h*w for all-reduced sums)
int bn_bwd_apply_n(const void* dA, long dA_ld, const void* z, long z_ld, const float* gamma, const float* scale,
                   const float* shift, const float* save_mean, const float* save_invstd, const float* dgamma,
                   const float* dbeta, long count, int n, int h, int w, int c, int dtype, int leaky, int upsample2x,
                   int dilate2x, void* dz, long dz_ld, void* stream) {
  YB_BN_COMMON_CHECK("bn_bwd_apply");
  YB_REQUIRE(dA && z && gamma && scale && shift && save_mean && save_invstd && dgamma && dbeta && dz,
             "bn_bwd_apply: null pointer");
  YB_REQUIRE(count >= (long)n * h * w, "bn_bwd_apply: count must cover the local rows");
  RowGeom g{(long)n * h * w, h, w, c};
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int grid, cpt;
  const StreamGeom sg = stream_geom(g.rows, c, &cpt, &grid);
  const int vec = aligned16({gamma, scale, shift, save_mean, save_invstd, dgamma, dbeta});
#define YB_APP_LAUNCH(T, CPT, R, BPS)                                                                                  \
  bn_bwd_apply_kernel<T, CPT, R, BPS><<<grid, 256, 0, st>>>((const T*)dA, dA_ld, (const T*)z, z_ld, gamma, scale,      \
                                                            shift, save_mean, save_invstd, dgamma, dbeta, g, sg, leaky, \
                                                            upsample2x, dilate2x, vec, (float)count, (T*)dz, dz_ld)
  YB_BN_DTYPES(YB_APP_LAUNCH)
#undef YB_APP_LAUNCH
  YB_CUDA(cudaGetLastError());
  return YB_OK;
}
}  // namespace yb

extern "C" int yb_bn_bwd_apply(const void* dA, long dA_ld, const void* z, long z_ld, const float* gamma,
                               const float* scale, const float* shift, const float* save_mean,
                               const float* save_invstd, const float* dgamma, const float* dbeta, int n, int h, int w,
                               int c, int dtype, int leaky, int upsample2x, int dilate2x, void* dz, long dz_ld,
                               void* stream) {
  return bn_bwd_apply_n(dA, dA_ld, z, z_ld, gamma, scale, shift, save_mean, save_invstd, dgamma, dbeta, (long)n * h * w,
                        n, h, w, c, dtype, leaky, upsample2x, dilate2x, dz, dz_ld, stream);
}

extern "C" int yb_col_stats(const void* x, long ld, long rows, int c, int dtype, float* sum, float* sqsum, void* stream);
extern "C" int yb_col_sum(const void* x, long ld, long rows, int c, int dtype, float* out, void* stream) {
  return yb_col_stats(x, ld, rows, c, dtype, out, nullptr, stream);
}
extern "C" int yb_col_stats(const void* x, long ld, long rows, int c, int dtype, float* out, float* out_sq, void* stream) {
  YB_REQUIRE(x && out && rows > 0 && c > 0, "col_sum: bad argument");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  YB_CUDA(cudaMemsetAsync(out, 0, c * 4, st));
  if (out_sq) YB_CUDA(cudaMemsetAsync(out_sq, 0, c * 4, st));
  const int gy = ceil_div(c, 32);
  long slabs = (long)num_sms() * 8 / gy;
  if (slabs < 1) slabs = 1;
  long rpb = (rows + slabs - 1) / slabs;
  if (rpb < 32) rpb = 32;
  dim3 grid(ceil_div(rows, rpb), gy), block(32, 8);
  if (dtype == YB_F16) col_sum_kernel<__half><<<grid, block, 0, st>>>((const __half*)x, ld, rows, c, rpb, out, out_sq);
  else if (dtype == YB_BF16) col_sum_kernel<__nv_bfloat16><<<grid, block, 0, st>>>((const __nv_bfloat16*)x, ld, rows, c, rpb, out, out_sq);
  else if (dtype == YB_F32) col_sum_kernel<float><<<grid, block, 0, st>>>((const float*)x, ld, rows, c, rpb, out, out_sq);
  else { set_error("col_sum: bad dtype"); return YB_ERR_UNSUPPORTED; }
  YB_CUDA(cudaGetLastError());
  return YB_OK;
}
