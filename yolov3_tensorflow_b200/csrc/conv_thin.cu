// Direct 3x3 convolution for the THIN layers at the top of Darknet-53 (the stem 3->32 and the Cin = 32
// layers darknet53_body/Conv_1, Conv_3; utils/layer_utils.py:35-36,27): they are HBM-bound (12-64 B in,
// 64-128 B out per pixel, <= 1.6 GFLOP/img) and the implicit-GEMM path is a poor fit for them — with 32
// input channels an im2col row is 64 B, which halves the TMA line rate, and every input pixel is re-fetched
// 9x from L2.  Here every input pixel is
// read from global memory ONCE per tile into a shared-memory halo tile, the (tiny) weight matrix stays
// resident in shared memory, and the 9-tap reduction runs out of shared memory on the warp-level tensor
// path (ldmatrix + mma.sync m16n8k16, fp32 accumulate) — per-warp gathers through ldmatrix row addresses
// need no im2col copy at all.  Epilogue: scale/shift + leaky (+ residual), staged through shared memory so
// that global stores are full 128-byte rows.
#include "common.cuh"

namespace yb {

static constexpr int TH = 8, TW = 16;          // output pixels per CTA tile: 8 rows x 16 cols = 128
static constexpr int THIN_THREADS = 128;       // 4 warps, each 2 output rows (two m16 tiles) x all channels

struct ThinParams {
  const void* x;        // input activation (16-bit NHWC) or float32 image for the stem
  long x_ld;            // elements between input pixels
  const void* wt;       // packed weights [cout_pad][9*cin] 16-bit (layers) / OHWI float32 [32][27] (stem)
  const float* scale;
  const float* shift;
  const void* res;      // nullable, 16-bit [n, ho, wo, res_ld]
  long res_ld;
  void* out;            // 16-bit [n, ho, wo, out_ld]
  long out_ld;
  int n, h, w;          // input spatial size
  int ho, wo;           // output spatial size
  int tiles_y, tiles_x, num_tiles;
  int leaky;
  int dbg;              // timing experiments (YB_STEM_DBG bitmask): 1 no halo load, 2 no im2col, 4 no MMA, 8 no stores
  float* stat_sum;      // stem only, nullable: per-channel sum / sum of squares of the STORED (16-bit) outputs, accumulated
  float* stat_sqsum;    //   (the BN batch statistics of the training forward: no separate pass over the 354 MB tensor)
};

__device__ __forceinline__ void cp_async16(void* dst, const void* src, int src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(dst)), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }
__device__ __forceinline__ void ldmatrix_x4(uint32_t (&r)[4], const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(smem_u32(p)));
}
template <typename T>
__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1);
template <>
__device__ __forceinline__ void mma16816<__half>(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
template <>
__device__ __forceinline__ void mma16816<__nv_bfloat16>(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// CIN = 32 (layers) ; STEM: CIN = 3 float32 image, K padded 27 -> 32.
// SPLIT (stem only; the training forward): split-precision operands, K = 96 = [x_hi | x_lo | x_hi] . [w_hi ; w_hi ; w_lo]
// with v_hi = T(v), v_lo = T(v - v_hi): the products keep ~16 bits of the float32 image and weights (only lo x lo,
// 2^-16 relative for bf16, is dropped), so the raw stem output feeding the batch statistics matches a float32
// convolution like the reference's (model.py:35, utils/layer_utils.py:35) instead of one on operands rounded to 8 bits.
template <typename T, int COUT, int STRIDE, bool STEM, bool SPLIT = false>
struct ThinCfg {
  static constexpr int CIN = STEM ? 3 : 32;
  static constexpr int K = STEM ? (SPLIT ? 96 : 32) : 9 * 32;   // GEMM K
  static constexpr int HH = TH * STRIDE + 2, HW = TW * STRIDE + 2;   // halo tile
  static constexpr int PIX_PITCH = STEM ? 0 : (32 * 2 + 16);    // bytes per halo pixel (padded: conflict-free ldmatrix)
  static constexpr int HALO_BYTES = STEM ? HH * HW * 3 * 4 : HH * HW * PIX_PITCH;
  static constexpr int W_PITCH = K * 2 + 16;                    // bytes per weight row (one output channel)
  static constexpr int W_BYTES = COUT * W_PITCH;
  static constexpr int A_PITCH = (STEM ? K : 32) * 2 + 16;      // stem only: im2col'd [128][K] tile
  static constexpr int A_BYTES = STEM ? 128 * A_PITCH : 0;
  static constexpr int O_PITCH = COUT * 2 + 16;                 // output staging [128 px][COUT]
  static constexpr int O_BYTES = 128 * O_PITCH;
  // the output staging tile reuses the halo tile's storage (the halo is dead once the MMAs are done)
  static constexpr int HALO_OR_OUT = (HALO_BYTES > O_BYTES ? HALO_BYTES : O_BYTES);
  static constexpr int SMEM = ((HALO_OR_OUT + 127) / 128) * 128 + W_BYTES + A_BYTES + 128;
};

template <typename T, int COUT, int STRIDE, bool STEM, bool SPLIT = false>
__global__ void __launch_bounds__(THIN_THREADS)
conv_thin_kernel(const ThinParams p) {
  using C = ThinCfg<T, COUT, STRIDE, STEM, SPLIT>;
  static_assert(!SPLIT || STEM, "split-precision operands exist for the stem only");
  extern __shared__ __align__(128) uint8_t tsm[];
  uint8_t* s_halo = tsm;
  uint8_t* s_w = tsm + ((C::HALO_OR_OUT + 127) / 128) * 128;
  uint8_t* s_a = s_w + C::W_BYTES;
  uint8_t* s_o = tsm;                                             // aliases s_halo
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  // ---- weights: resident for the whole (persistent) CTA ----
  if (STEM) {
    const float* wf = static_cast<const float*>(p.wt);          // [COUT][27]
    for (int i = tid; i < COUT * 32; i += THIN_THREADS) {
      const int co = i >> 5, k = i & 31;
      const float wv = k < 27 ? wf[co * 27 + k] : 0.f;
      T* wrow = reinterpret_cast<T*>(s_w + co * C::W_PITCH);
      const T hi = static_cast<T>(wv);
      wrow[k] = hi;
      if (SPLIT) { wrow[32 + k] = hi; wrow[64 + k] = static_cast<T>(wv - static_cast<float>(hi)); }
    }
  } else {
    const uint8_t* wg = static_cast<const uint8_t*>(p.wt);      // [cout_pad][288] 16-bit
    constexpr int CH = C::K * 2 / 16;                           // 16-byte chunks per row
    for (int i = tid; i < COUT * CH; i += THIN_THREADS) {
      const int co = i / CH, ch = i - co * CH;
      cp_async16(s_w + co * C::W_PITCH + ch * 16, wg + ((long)co * C::K * 2) + ch * 16, 16);
    }
  }

  // stem: the NEXT tile's halo (float32 image) is fetched into registers while the current tile is processed — a
  // tile's 540 scalar loads would otherwise be issued and awaited serially
  constexpr int HN = STEM ? C::HH * C::HW * 3 : 1;
  constexpr int NL = (HN + THIN_THREADS - 1) / THIN_THREADS;
  float pre[NL];
  auto fetch_halo = [&](int tile) {
    const int tx = tile % p.tiles_x;
    const int ty = (tile / p.tiles_x) % p.tiles_y;
    const int img = tile / (p.tiles_x * p.tiles_y);
    const int iy0 = ty * TH * STRIDE - 1, ix0 = tx * TW * STRIDE - 1;
    const float* xin = static_cast<const float*>(p.x) + (long)img * p.h * p.w * 3;
#pragma unroll
    for (int k = 0; k < NL; ++k) {
      const int i = tid + k * THIN_THREADS;
      const int c = i % 3, px = (i / 3) % C::HW, py = i / (3 * C::HW);
      const int gy = iy0 + py, gx = ix0 + px;
      pre[k] = (i < HN && gy >= 0 && gy < p.h && gx >= 0 && gx < p.w) ? __ldg(xin + ((long)gy * p.w + gx) * 3 + c) : 0.f;
    }
  };
  if (STEM && (int)blockIdx.x < p.num_tiles && !(p.dbg & 1)) fetch_halo(blockIdx.x);
  float st_s = 0.f, st_q = 0.f;   // stem statistics: thread = (warp: 32-pixel quarter of every tile, lane: channel)

  for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
    const int tx = tile % p.tiles_x;
    const int ty = (tile / p.tiles_x) % p.tiles_y;
    const int img = tile / (p.tiles_x * p.tiles_y);
    const int oy0 = ty * TH, ox0 = tx * TW;
    const int iy0 = oy0 * STRIDE - 1, ix0 = ox0 * STRIDE - 1;
    __syncthreads();                                            // previous tile done with s_halo / s_o
    // ---- halo tile ----
    if (STEM) {
      float* hf = reinterpret_cast<float*>(s_halo);
      if (!(p.dbg & 1)) {
#pragma unroll
        for (int k = 0; k < NL; ++k) {
          const int i = tid + k * THIN_THREADS;
          if (i < HN) hf[i] = pre[k];
        }
        if (tile + (int)gridDim.x < p.num_tiles) fetch_halo(tile + gridDim.x);
      }
    } else {
      const T* xin = static_cast<const T*>(p.x) + (long)img * p.h * p.w * p.x_ld;
      for (int i = tid; i < C::HH * C::HW * 4; i += THIN_THREADS) {
        const int ch = i & 3, px = (i >> 2) % C::HW, py = (i >> 2) / C::HW;
        const int gy = iy0 + py, gx = ix0 + px;
        const bool ok = gy >= 0 && gy < p.h && gx >= 0 && gx < p.w;
        const T* src = ok ? xin + ((long)gy * p.w + gx) * p.x_ld + ch * 8 : xin;
        cp_async16(s_halo + (py * C::HW + px) * C::PIX_PITCH + ch * 16, src, ok ? 16 : 0);   // zero-fill outside
      }
    }
    cp_async_wait_all();
    __syncthreads();
    if (STEM && !(p.dbg & 2)) {
      // im2col of the thread's pixel: 27 taps -> one 32-wide fp16 row
      const float* hf = reinterpret_cast<const float*>(s_halo);
      const int py = tid / TW, px = tid % TW;
      float pv[32];
#pragma unroll
      for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int s = 0; s < 3; ++s)
#pragma unroll
          for (int c = 0; c < 3; ++c) pv[(r * 3 + s) * 3 + c] = hf[((py + r) * C::HW + (px + s)) * 3 + c];
#pragma unroll
      for (int k = 27; k < 32; ++k) pv[k] = 0.f;
      uint4* arow = reinterpret_cast<uint4*>(s_a + tid * C::A_PITCH);   // 16-byte aligned rows (pitch = 2 K + 16 bytes)
#pragma unroll
      for (int j = 0; j < 4; ++j) {                                     // four 128-bit stores instead of 32 16-bit ones
        uint4 u;
        u.x = Pack2<T>::pack(pv[8 * j + 0], pv[8 * j + 1]); u.y = Pack2<T>::pack(pv[8 * j + 2], pv[8 * j + 3]);
        u.z = Pack2<T>::pack(pv[8 * j + 4], pv[8 * j + 5]); u.w = Pack2<T>::pack(pv[8 * j + 6], pv[8 * j + 7]);
        arow[j] = u;
        if (SPLIT) {                                                    // [x_hi | x_lo | x_hi]
          arow[8 + j] = u;
          float lo[8];
          float2 f;
          f = Pack2<T>::unpack(u.x); lo[0] = pv[8 * j + 0] - f.x; lo[1] = pv[8 * j + 1] - f.y;
          f = Pack2<T>::unpack(u.y); lo[2] = pv[8 * j + 2] - f.x; lo[3] = pv[8 * j + 3] - f.y;
          f = Pack2<T>::unpack(u.z); lo[4] = pv[8 * j + 4] - f.x; lo[5] = pv[8 * j + 5] - f.y;
          f = Pack2<T>::unpack(u.w); lo[6] = pv[8 * j + 6] - f.x; lo[7] = pv[8 * j + 7] - f.y;
          uint4 l;
          l.x = Pack2<T>::pack(lo[0], lo[1]); l.y = Pack2<T>::pack(lo[2], lo[3]);
          l.z = Pack2<T>::pack(lo[4], lo[5]); l.w = Pack2<T>::pack(lo[6], lo[7]);
          arow[4 + j] = l;
        }
      }
    }
    if (STEM) __syncthreads();
    // ---- main loop: each warp computes 2 output rows (2 x m16) x COUT ----
    constexpr int NT = COUT / 8;                                // n8 tiles
    float acc[2][NT][4];
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
      for (int nj = 0; nj < NT; ++nj)
#pragma unroll
        for (int q = 0; q < 4; ++q) acc[mi][nj][q] = 0.f;
    constexpr int KSTEPS = C::K / 16;
#pragma unroll 1
    for (int ks = 0; ks < ((STEM && (p.dbg & 4)) ? 0 : KSTEPS); ++ks) {
      uint32_t a[2][4];
#pragma unroll
      for (int mi = 0; mi < 2; ++mi) {
        const int y = warp * 2 + mi, x = lane & 15, kh = lane >> 4;          // row of the m16 tile / k half
        const uint8_t* ap;
        if (STEM) {
          ap = s_a + (y * TW + x) * C::A_PITCH + (ks * 16 + kh * 8) * 2;
        } else {
          const int tap = ks >> 1, kc = ks & 1;
          const int r = tap / 3, s = tap - r * 3;
          ap = s_halo + ((y * STRIDE + r) * C::HW + (x * STRIDE + s)) * C::PIX_PITCH + (kc * 16 + kh * 8) * 2;
        }
        ldmatrix_x4(a[mi], ap);
      }
#pragma unroll
      for (int nb = 0; nb < NT / 2; ++nb) {
        // 16 output channels x k16: matrices (n0-7,k0-7), (n0-7,k8-15), (n8-15,k0-7), (n8-15,k8-15)
        uint32_t b[4];
        const int nrow = nb * 16 + (lane & 7) + ((lane >> 4) & 1) * 8;
        const int kof = ks * 16 + ((lane >> 3) & 1) * 8;
        ldmatrix_x4(b, s_w + nrow * C::W_PITCH + kof * 2);
#pragma unroll
        for (int mi = 0; mi < 2; ++mi) {
          mma16816<T>(acc[mi][2 * nb], a[mi], b[0], b[1]);
          mma16816<T>(acc[mi][2 * nb + 1], a[mi], b[2], b[3]);
        }
      }
    }
    __syncthreads();                                            // every warp is done reading the halo tile (s_o aliases it)
    // ---- epilogue: scale/shift/leaky -> shared staging ----
#pragma unroll
    for (int mi = 0; mi < 2; ++mi) {
      const int y = warp * 2 + mi;
#pragma unroll
      for (int nj = 0; nj < NT; ++nj) {
        const int c0 = nj * 8 + (lane & 3) * 2;
        const float sc0 = __ldg(p.scale + c0), sc1 = __ldg(p.scale + c0 + 1);
        const float sh0 = __ldg(p.shift + c0), sh1 = __ldg(p.shift + c0 + 1);
#pragma unroll
        for (int hrow = 0; hrow < 2; ++hrow) {
          const int x = (lane >> 2) + hrow * 8;
          float v0 = fmaf(acc[mi][nj][hrow * 2 + 0], sc0, sh0);
          float v1 = fmaf(acc[mi][nj][hrow * 2 + 1], sc1, sh1);
          if (p.leaky) { v0 = leaky01(v0); v1 = leaky01(v1); }
          if (p.res == nullptr) {
            *reinterpret_cast<uint32_t*>(s_o + (y * TW + x) * C::O_PITCH + c0 * 2) = Pack2<T>::pack(v0, v1);
          } else {   // keep fp32 precision until the residual is added: stage as two halves of a float2? no room -> add here
            const int oy = oy0 + y, ox = ox0 + x;
            if (oy < p.ho && ox < p.wo) {
              const uint32_t ru = *reinterpret_cast<const uint32_t*>(static_cast<const T*>(p.res) +
                                                                    (((long)img * p.ho + oy) * p.wo + ox) * p.res_ld + c0);
              const float2 rf = Pack2<T>::unpack(ru);
              v0 += rf.x; v1 += rf.y;
            }
            *reinterpret_cast<uint32_t*>(s_o + (y * TW + x) * C::O_PITCH + c0 * 2) = Pack2<T>::pack(v0, v1);
          }
        }
      }
    }
    __syncthreads();
    if (STEM && p.stat_sum != nullptr) {
      // column sums over the staged tile (the values exactly as stored): a warp's lanes read one pixel's 32 channels
#pragma unroll 4
      for (int i = 0; i < 32; ++i) {
        const int px = warp * 32 + i;
        if (oy0 + px / TW < p.ho && ox0 + px % TW < p.wo) {
          const float v = static_cast<float>(reinterpret_cast<const T*>(s_o + px * C::O_PITCH)[lane]);
          st_s += v;
          st_q = fmaf(v, v, st_q);
        }
      }
    }
    // ---- coalesced copy-out: one 16-byte chunk per thread-iteration, full rows of COUT*2 bytes ----
    constexpr int OCH = COUT * 2 / 16;
    for (int i = tid; i < 128 * OCH; i += THIN_THREADS) {
      const int px = i / OCH, ch = i - px * OCH;
      const int oy = oy0 + px / TW, ox = ox0 + px % TW;
      if (oy < p.ho && ox < p.wo && !(STEM && (p.dbg & 8))) {
        const uint4 v = *reinterpret_cast<const uint4*>(s_o + px * C::O_PITCH + ch * 16);
        *reinterpret_cast<uint4*>(static_cast<T*>(p.out) + (((long)img * p.ho + oy) * p.wo + ox) * p.out_ld + ch * 8) = v;
      }
    }
  }
  cp_async_wait_all();
  if (STEM && p.stat_sum != nullptr) {          // 2 x 128 atomics per persistent CTA
    atomicAdd(p.stat_sum + lane, st_s);
    atomicAdd(p.stat_sqsum + lane, st_q);
  }
}

__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t (&r)[4], const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(smem_u32(p)));
}

// Weight gradient of the stem (float32 image, 3 -> 32 channels, utils/layer_utils.py:35):
//   dW[co, k] = sum_p dz[p, co] * patch[p, k],   k = (r*3+s)*3+c  (27, padded to 32)
// on the warp-level tensor path: D[32 co x 32 k] += dz^T[32 x 128 px] * patch[128 px x 32] per 8x16-pixel tile.  Both
// operands are stored pixel-major in shared memory and read with ldmatrix.trans.  The image stays float32-exact:
// every patch value is split into a 16-bit head and a 16-bit remainder (x = hi + lo) and both products are
// accumulated, so the result matches a float32 convolution-backward to ~1e-5.
// Each of the 4 warps reduces 32 of the tile's 128 pixels; accumulators live in registers across all tiles of the
// persistent CTA and are combined through shared memory at the end (864 global atomics per CTA).
template <typename T>
__global__ void __launch_bounds__(THIN_THREADS)
stem_wgrad_tc_kernel(const float* __restrict__ x, const T* __restrict__ dz, int n, int h, int w, int tiles_y,
                     int tiles_x, int num_tiles, float* __restrict__ dw) {
  constexpr int HH = TH + 2, HW = TW + 2;
  constexpr int PITCH = 32 * 2 + 16;                      // bytes per pixel row of the 16-bit tiles
  __shared__ __align__(16) float s_halo[HH * HW * 3];
  __shared__ __align__(16) uint8_t s_hi[128 * PITCH], s_lo[128 * PITCH], s_dz[128 * PITCH];
  __shared__ float s_acc[32 * 32];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  for (int i = tid; i < 32 * 32; i += THIN_THREADS) s_acc[i] = 0.f;
  float acc[2][4][4];
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int nj = 0; nj < 4; ++nj)
#pragma unroll
      for (int q = 0; q < 4; ++q) acc[mi][nj][q] = 0.f;

  constexpr int HN = HH * HW * 3;
  constexpr int NL = (HN + THIN_THREADS - 1) / THIN_THREADS;
  float pre[NL];
  auto fetch_halo = [&](int tile) {
    const int tx = tile % tiles_x;
    const int ty = (tile / tiles_x) % tiles_y;
    const int img = tile / (tiles_x * tiles_y);
    const float* xin = x + (long)img * h * w * 3;
#pragma unroll
    for (int k = 0; k < NL; ++k) {
      const int i = tid + k * THIN_THREADS;
      const int c = i % 3, px = (i / 3) % HW, py = i / (3 * HW);
      const int gy = ty * TH - 1 + py, gx = tx * TW - 1 + px;
      pre[k] = (i < HN && gy >= 0 && gy < h && gx >= 0 && gx < w) ? __ldg(xin + ((long)gy * w + gx) * 3 + c) : 0.f;
    }
  };
  if ((int)blockIdx.x < num_tiles) fetch_halo(blockIdx.x);

  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const int tx = tile % tiles_x;
    const int ty = (tile / tiles_x) % tiles_y;
    const int img = tile / (tiles_x * tiles_y);
    const int oy0 = ty * TH, ox0 = tx * TW;
    __syncthreads();                                      // previous tile's fragments are consumed
    // dz tile: 128 pixels x 64 bytes (zero outside the image)
    for (int i = tid; i < 128 * 4; i += THIN_THREADS) {
      const int px = i >> 2, ch = i & 3;
      const int oy = oy0 + px / TW, ox = ox0 + px % TW;
      const bool ok = oy < h && ox < w;
      const T* src = ok ? dz + (((long)img * h + oy) * w + ox) * 32 + ch * 8 : dz;
      cp_async16(s_dz + px * PITCH + ch * 16, src, ok ? 16 : 0);
    }
#pragma unroll
    for (int k = 0; k < NL; ++k) {
      const int i = tid + k * THIN_THREADS;
      if (i < HN) s_halo[i] = pre[k];
    }
    if (tile + (int)gridDim.x < num_tiles) fetch_halo(tile + gridDim.x);   // next tile's image halo, in flight during this tile
    __syncthreads();
    {   // im2col of the thread's pixel, split into head + remainder
      const int py = tid / TW, px = tid % TW;
      uint32_t* hi = reinterpret_cast<uint32_t*>(s_hi + tid * PITCH);
      uint32_t* lo = reinterpret_cast<uint32_t*>(s_lo + tid * PITCH);
      float v[32];
#pragma unroll
      for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int s2 = 0; s2 < 3; ++s2)
#pragma unroll
          for (int c = 0; c < 3; ++c) v[(r * 3 + s2) * 3 + c] = s_halo[((py + r) * HW + (px + s2)) * 3 + c];
#pragma unroll
      for (int k = 27; k < 32; ++k) v[k] = 0.f;
#pragma unroll
      for (int j = 0; j < 4; ++j) {                       // 128-bit stores (80-byte row pitch keeps 16-byte alignment)
        uint32_t hq[4], lq[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int k = 8 * j + 2 * e;
          hq[e] = Pack2<T>::pack(v[k], v[k + 1]);
          const float2 hf = Pack2<T>::unpack(hq[e]);
          lq[e] = Pack2<T>::pack(v[k] - hf.x, v[k + 1] - hf.y);
        }
        reinterpret_cast<uint4*>(hi)[j] = make_uint4(hq[0], hq[1], hq[2], hq[3]);
        reinterpret_cast<uint4*>(lo)[j] = make_uint4(lq[0], lq[1], lq[2], lq[3]);
      }
    }
    cp_async_wait_all();
    __syncthreads();
    // warp `warp` reduces pixels [32*warp, 32*warp + 32): two k16 steps
#pragma unroll
    for (int ks = 0; ks < 2; ++ks) {
      const int p0 = warp * 32 + ks * 16;
      const int mi_ = lane >> 3, rr = lane & 7;
      uint32_t a[2][4];
#pragma unroll
      for (int mi = 0; mi < 2; ++mi)   // matrices: (co 0-7, px 0-7), (co 8-15, px 0-7), (co 0-7, px 8-15), (co 8-15, px 8-15)
        ldmatrix_x4_trans(a[mi], s_dz + (p0 + (mi_ >> 1) * 8 + rr) * PITCH + (mi * 16 + (mi_ & 1) * 8) * 2);
#pragma unroll
      for (int part = 0; part < 2; ++part) {
        const uint8_t* bt = part == 0 ? s_hi : s_lo;
#pragma unroll
        for (int nb = 0; nb < 2; ++nb) {   // matrices: (px 0-7, k 0-7), (px 8-15, k 0-7), (px 0-7, k 8-15), (px 8-15, k 8-15)
          uint32_t b[4];
          ldmatrix_x4_trans(b, bt + (p0 + (mi_ & 1) * 8 + rr) * PITCH + (nb * 16 + (mi_ >> 1) * 8) * 2);
#pragma unroll
          for (int mi = 0; mi < 2; ++mi) {
            mma16816<T>(acc[mi][2 * nb], a[mi], b[0], b[1]);
            mma16816<T>(acc[mi][2 * nb + 1], a[mi], b[2], b[3]);
          }
        }
      }
    }
  }
  __syncthreads();
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int nj = 0; nj < 4; ++nj)
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int co = mi * 16 + (lane >> 2) + (q >> 1) * 8;
        const int k = nj * 8 + (lane & 3) * 2 + (q & 1);
        atomicAdd(&s_acc[co * 32 + k], acc[mi][nj][q]);
      }
  __syncthreads();
  for (int i = tid; i < 32 * 27; i += THIN_THREADS) {
    const int co = i / 27, k = i - co * 27;
    atomicAdd(dw + i, s_acc[co * 32 + k]);
  }
}

// One conv_thin_kernel instantiation: the type thin_kernel_for passes to its functor
template <typename T, int COUT, int STRIDE, bool STEM, bool SPLIT = false>
struct ThinKernel {
  using C = ThinCfg<T, COUT, STRIDE, STEM, SPLIT>;
  static constexpr auto kernel = conv_thin_kernel<T, COUT, STRIDE, STEM, SPLIT>;
};

// The instantiation a conv_thin_kernel launch needs.  Host only: ThinParams is the kernel's by-value parameter.
struct ThinKey {
  int dtype;           // yb_dtype of the 16-bit operands and output
  int cout, stride;
  bool stem, split;    // the stem (float32 image, 3 input channels); split-precision operands (stem only)
};

static int no_thin_kernel(const ThinKey& k) {
  set_error("conv_thin: no kernel for dtype %d, cout=%d stride=%d, stem %d, split operands %d", k.dtype, k.cout, k.stride,
            (int)k.stem, (int)k.split);
  return YB_ERR_UNSUPPORTED;
}

template <typename T, typename F>
static int thin_kernel_type(const ThinKey& k, F& f) {
  if (k.stem) {
    if (k.cout == 32 && k.stride == 1) return k.split ? f(ThinKernel<T, 32, 1, true, true>()) : f(ThinKernel<T, 32, 1, true>());
    return no_thin_kernel(k);
  }
  if (k.split) return no_thin_kernel(k);
  if (k.cout == 64 && k.stride == 1) return f(ThinKernel<T, 64, 1, false>());
  if (k.cout == 64 && k.stride == 2) return f(ThinKernel<T, 64, 2, false>());
  if (k.cout == 32 && k.stride == 1) return f(ThinKernel<T, 32, 1, false>());
  if (k.cout == 32 && k.stride == 2) return f(ThinKernel<T, 32, 2, false>());
  return no_thin_kernel(k);
}

// The instantiation table: every conv_thin_kernel that exists is named here and nowhere else.  Calls
// f(ThinKernel<...>()) with the instantiation of k and returns what f returns, or YB_ERR_UNSUPPORTED when there is none.
template <typename F>
static int thin_kernel_for(const ThinKey& k, F&& f) {
  if (k.dtype == YB_F16) return thin_kernel_type<__half>(k, f);
  if (k.dtype == YB_BF16) return thin_kernel_type<__nv_bfloat16>(k, f);
  return no_thin_kernel(k);
}

template <typename K>
static int thin_launch_kernel(const ThinParams& p, cudaStream_t st) {
  static DeviceOnce once;
  auto kern = K::kernel;
  { const int rc = ensure_smem_attr(once, reinterpret_cast<const void*>(kern), K::C::SMEM); if (rc) return rc; }
  int per_sm = 227 * 1024 / (K::C::SMEM + 1024);
  if (per_sm < 1) per_sm = 1;
  if (per_sm > 8) per_sm = 8;
  const int grid = p.num_tiles < num_sms() * per_sm ? p.num_tiles : num_sms() * per_sm;
  kern<<<grid, THIN_THREADS, K::C::SMEM, st>>>(p);
  YB_CUDA(cudaGetLastError());
  return YB_OK;
}

static int thin_launch(const ThinKey& key, const ThinParams& p, cudaStream_t st) {
  return thin_kernel_for(key, [&](auto k) -> int { return thin_launch_kernel<decltype(k)>(p, st); });
}

}  // namespace yb

using namespace yb;

// 3x3 conv, cin = 32, cout in {32, 64}, stride 1|2, no BN statistics (inference epilogue).
extern "C" int yb_conv3x3_thin_fwd(const yb_conv_desc* d, const void* x, const void* w_packed, const float* scale,
                                   const float* shift, const void* res, void* out, void* stream) {
  YB_REQUIRE(d && x && w_packed && scale && shift && out, "conv_thin: null pointer");
  YB_REQUIRE(d->ksize == 3 && d->cin == 32 && (d->cout == 64 || d->cout == 32) && (d->stride == 1 || d->stride == 2),
             "conv_thin: supports 3x3, cin=32, cout in {32,64}, stride 1|2 (got k=%d cin=%d cout=%d s=%d)", d->ksize, d->cin,
             d->cout, d->stride);
  YB_REQUIRE(d->dtype == YB_F16 || d->dtype == YB_BF16, "conv_thin: dtype must be f16 or bf16");
  YB_REQUIRE(!d->out_fp32 && !d->upsample2x, "conv_thin: 16-bit, non-upsampled outputs only");
  YB_REQUIRE(d->in_ld % 8 == 0 && d->out_ld % 8 == 0 && (!res || d->res_ld % 2 == 0), "conv_thin: bad leading dimensions");
  ThinParams p;
  p.x = x; p.x_ld = d->in_ld; p.wt = w_packed; p.scale = scale; p.shift = shift; p.res = res; p.res_ld = d->res_ld;
  p.out = out; p.out_ld = d->out_ld; p.n = d->n; p.h = d->h; p.w = d->w;
  p.ho = d->h / d->stride; p.wo = d->w / d->stride;
  p.tiles_y = ceil_div(p.ho, TH); p.tiles_x = ceil_div(p.wo, TW);
  p.num_tiles = p.tiles_x * p.tiles_y * d->n;
  p.leaky = d->leaky; p.dbg = 0; p.stat_sum = nullptr; p.stat_sqsum = nullptr;
  return thin_launch(ThinKey{d->dtype, d->cout, d->stride, false, false}, p, static_cast<cudaStream_t>(stream));
}

// Stem on the warp-level tensor path: float32 image [n,h,w,3] -> 16-bit [n,h,w,32]; w_ohwi float32 [32][27].
// stat_sum / stat_sqsum (both or neither; zeroed by the caller): the kernel also ACCUMULATES the per-channel sum and sum
// of squares of the stored outputs — the batch statistics slim.batch_norm(is_training=True) needs (model.py:35-41).
extern "C" int yb_stem_conv_fwd_tc_stats(const float* x, const float* w_ohwi, const float* scale, const float* shift,
                                         int n, int h, int w, int dtype, int leaky, void* out, float* stat_sum,
                                         float* stat_sqsum, void* stream) {
  YB_REQUIRE(x && w_ohwi && scale && shift && out && n > 0 && h > 0 && w > 0, "stem_tc: bad argument");
  YB_REQUIRE((stat_sum == nullptr) == (stat_sqsum == nullptr), "stem_tc: stat_sum/stat_sqsum must both be given");
  ThinParams p;
  p.x = x; p.x_ld = 3; p.wt = w_ohwi; p.scale = scale; p.shift = shift; p.res = nullptr; p.res_ld = 0;
  p.out = out; p.out_ld = 32; p.n = n; p.h = h; p.w = w; p.ho = h; p.wo = w;
  p.tiles_y = ceil_div(h, TH); p.tiles_x = ceil_div(w, TW);
  p.num_tiles = p.tiles_x * p.tiles_y * n;
  p.leaky = leaky;
  p.dbg = opt_int("YB_STEM_DBG", 0);
  p.stat_sum = stat_sum; p.stat_sqsum = stat_sqsum;
  // the statistics-producing form is the training forward: split-precision operands (YB_STEM_SPLIT=0: plain 16-bit)
  const bool split = stat_sum != nullptr && opt("YB_STEM_SPLIT")[0] != '0';
  return thin_launch(ThinKey{dtype, 32, 1, true, split}, p, static_cast<cudaStream_t>(stream));
}
extern "C" int yb_stem_conv_fwd_tc(const float* x, const float* w_ohwi, const float* scale, const float* shift, int n,
                                   int h, int w, int dtype, int leaky, void* out, void* stream) {
  return yb_stem_conv_fwd_tc_stats(x, w_ohwi, scale, shift, n, h, w, dtype, leaky, out, nullptr, nullptr, stream);
}

// Stem weight gradient on the warp-level tensor path (float32 image split into 16-bit head + remainder).
extern "C" int yb_stem_conv_wgrad_tc(const float* x, const void* dz, int dtype, int n, int h, int w, float* dw,
                                     void* stream) {
  YB_REQUIRE(x && dz && dw && n > 0 && h > 0 && w > 0, "stem_wgrad_tc: bad argument");
  YB_REQUIRE(dtype == YB_F16 || dtype == YB_BF16, "stem_wgrad_tc: dtype must be f16 or bf16");
  const int tiles_y = ceil_div(h, TH), tiles_x = ceil_div(w, TW);
  const int num_tiles = tiles_x * tiles_y * n;
  const int grid = num_tiles < num_sms() * 4 ? num_tiles : num_sms() * 4;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (dtype == YB_F16)
    stem_wgrad_tc_kernel<__half><<<grid, THIN_THREADS, 0, st>>>(x, static_cast<const __half*>(dz), n, h, w, tiles_y,
                                                               tiles_x, num_tiles, dw);
  else
    stem_wgrad_tc_kernel<__nv_bfloat16><<<grid, THIN_THREADS, 0, st>>>(x, static_cast<const __nv_bfloat16*>(dz), n, h,
                                                                      w, tiles_y, tiles_x, num_tiles, dw);
  YB_CUDA(cudaGetLastError());
  return YB_OK;
}
