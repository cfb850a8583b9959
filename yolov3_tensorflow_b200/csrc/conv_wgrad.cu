// Weight gradient of a conv as a tensor-core GEMM reduced over the output pixels:
//
//   dW[co, (r,s), ci] = sum_p  dz[p, co] * x[n(p), h(p)*stride + r - pad, w(p)*stride + s - pad, ci]
//
//   M = co (128 per tile, 64 per consumer warpgroup), N = ci chunk of one filter tap (BNW = 32..128), K = pixels.
//   A = dz^T   : 2D tiled TMA boxes {64 co x 64 pixels} -> smem rows = pixels, 128 B of co
//                per row: the canonical *MN-major* 128B-swizzled wgmma layout.
//   B = x_col^T: TMA im2col boxes {BCH channels x 64 pixels} of filter tap (r,s) — the same
//                zero-filled border/stride handling as the forward conv — also MN-major.
//   D = fp32 in registers (wgmma); every CTA reduces one pixel range (split-K) of one output tile and
//       adds it into the fp32 gradient with vector atomics.
//   A CTA accumulates TP filter taps at once (one kernel row of a 3x3 filter): the dz tile is loaded once per TP taps
//   instead of once per tap, which keeps the large early layers, whose dz + x exceed the L2, off HBM speed.
// Replaces the wgrad half of TF autodiff for slim.conv2d (train.py:112).
#include <cudaTypedefs.h>

#include <type_traits>

#include "common.cuh"
#include "conv.cuh"
#include "wgmma.cuh"

namespace yb {

int make_tmap_2d(CUtensorMap* tm, const void* base, int dtype, long rows, long cols, long ld, int box_rows,
                 int box_cols, int weights);
int make_tmap_im2col_px(CUtensorMap* tm, const void* base, int dtype, int n, int h, int w, int c, long ld, int ksize,
                        int stride, int pad, int bk, int pixels);

static constexpr int WG_THREADS = 384;  // warpgroup 0: TMA producer (one thread), warpgroups 1, 2: 64 output channels each
static constexpr int WG_BKP = 64;     // pixels per pipeline stage
static constexpr int WG_BM = 128;     // output channels per tile

template <int BNW, int TP>
struct WCfg {
  static constexpr int BCH = BNW < 64 ? BNW : 64;            // channels per im2col box / swizzle row
  static constexpr int NB = BNW / BCH;                       // boxes per stage for B
  static constexpr int A_BYTES = WG_BM * WG_BKP * 2;         // 2 boxes of 64co x 64px
  static constexpr int B_BYTES = BNW * WG_BKP * 2;             // one tap
  static constexpr int STAGE_BYTES = A_BYTES + TP * B_BYTES;
  static constexpr int STAGES = (192 * 1024 / STAGE_BYTES) > 8 ? 8 : (192 * 1024 / STAGE_BYTES);
  static_assert(TP * BNW <= 192, "accumulators exceed the register budget");
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 + 256;
  static constexpr uint32_t B_ROW = BCH * 2;                 // bytes per pixel row of a B box (= its swizzle span)
};

template <typename T, int BNW, int TP>
__global__ void __launch_bounds__(WG_THREADS, 1)
conv_wgrad_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const WgradParams p) {
  using C = WCfg<BNW, TP>;
  extern __shared__ uint8_t smem_raw[];
  // 1024-byte alignment by POINTER ARITHMETIC on the __shared__ array (an integer round trip makes the pointer generic)
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* sA = smem;
  uint8_t* sB = smem + C::STAGES * C::A_BYTES;              // [stage][tap in group][B_BYTES]
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + C::STAGES * C::STAGE_BYTES);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + C::STAGES;                    // one arrive per consumer warp

  const int wg = threadIdx.x >> 7;
  // tile coordinates: blockIdx.x = pixel split, blockIdx.y = n tile (tap group, ci chunk), blockIdx.z = co tile
  const int tap0 = (blockIdx.y / p.n_chunks) * TP;
  const int ci0 = (blockIdx.y % p.n_chunks) * BNW;
  const int co0 = blockIdx.z * WG_BM;
  const int kb0 = blockIdx.x * p.kb_per_split;
  const int kb1 = min(kb0 + p.kb_per_split, p.num_kb);
  const int nkb = kb1 - kb0;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int i = 0; i < C::STAGES; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 8); }
    fence_barrier_init();
  }
  __syncthreads();
  if (nkb <= 0) return;

  if (wg == 0) {
    if (threadIdx.x == 0) {   // single-thread loop; the pixel coordinates of the 64-pixel block advance as counters
      int stage = 0; uint32_t phase = 0;
      const long pstart = (long)kb0 * WG_BKP;
      int q = (int)(pstart % p.wo), pp = (int)((pstart / p.wo) % p.ho), img = (int)(pstart / ((long)p.wo * p.ho));
      const bool two_a = co0 + 64 < p.cout;   // second 64-channel block exists (else its rows are masked anyway)
      const uint32_t tx_bytes = TP * C::B_BYTES + (two_a ? C::A_BYTES : C::A_BYTES / 2);
      for (int kb = kb0; kb < kb1; ++kb) {
        const long p0 = (long)kb * WG_BKP;
        mbar_wait(&empty_bar[stage], phase ^ 1);
        mbar_arrive_expect_tx(&full_bar[stage], tx_bytes);
        uint8_t* a = sA + stage * C::A_BYTES;
        if (p.a_dilated) {
          tma_load_im2col_4d(a, &tmA, &full_bar[stage], co0, 2 * q, 2 * pp, img, 0, 0);
          if (two_a) tma_load_im2col_4d(a + WG_BKP * 128, &tmA, &full_bar[stage], co0 + 64, 2 * q, 2 * pp, img, 0, 0);
        } else {
          tma_load_2d(a, &tmA, &full_bar[stage], co0, (int)p0);
          if (two_a) tma_load_2d(a + WG_BKP * 128, &tmA, &full_bar[stage], co0 + 64, (int)p0);
        }
#pragma unroll
        for (int t = 0; t < TP; ++t) {
          uint8_t* b = sB + (stage * TP + t) * C::B_BYTES;
          const int tap = tap0 + t;
          const int th = TP == 9 ? t / 3 : (TP == 3 ? tap0 / 3 : tap / p.ksize);
          const int tw = TP == 9 ? t % 3 : (TP == 3 ? t : tap % p.ksize);
#pragma unroll
          for (int j = 0; j < C::NB; ++j)
            tma_load_im2col_4d(b + j * WG_BKP * C::B_ROW, &tmB, &full_bar[stage], ci0 + j * C::BCH,
                               q * p.stride - p.pad, pp * p.stride - p.pad, img, (uint16_t)tw, (uint16_t)th);
        }
        q += WG_BKP;
        while (q >= p.wo) { q -= p.wo; if (++pp == p.ho) { pp = 0; ++img; } }
        if (++stage == C::STAGES) { stage = 0; phase ^= 1; }
      }
    }
  } else {
    // MMA: warpgroup cw owns output channels [co0 + 64 cw, co0 + 64 cw + 64) = A box cw.  Both operands are MN-major
    // (rows of the shared-memory tiles are pixels = K): A = dz^T one 64-channel swizzle atom wide, B = x_col^T.
    constexpr bool kBF16 = std::is_same<T, __nv_bfloat16>::value;
    const int cw = wg - 1;
    const int t = threadIdx.x & 127, lane = t & 31;
    float acc[TP][BNW / 2];
    int stage = 0, prev = 0; uint32_t phase = 0;
    for (int kb = kb0; kb < kb1; ++kb) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t a_addr = smem_u32(sA + stage * C::A_BYTES) + cw * WG_BKP * 128;
#pragma unroll
      for (int tt = 0; tt < TP; ++tt) wgmma_fence_operand(acc[tt]);
      wgmma_fence();
#pragma unroll
      for (int tt = 0; tt < TP; ++tt) {
        const uint32_t b_addr = smem_u32(sB + (stage * TP + tt) * C::B_BYTES);
#pragma unroll
        for (int k = 0; k < WG_BKP / 16; ++k) {
          const uint64_t adesc = make_smem_desc(a_addr + k * 16 * 128, WG_BKP * 128, 1024, 128);
          const uint64_t bdesc = make_smem_desc(b_addr + k * 16 * C::B_ROW, WG_BKP * C::B_ROW, 8 * C::B_ROW, C::B_ROW);
          Wgmma<BNW, kBF16, 1, 1>::mma(acc[tt], adesc, bdesc, (kb > kb0 || k > 0) ? 1 : 0);
        }
      }
      wgmma_commit();
#pragma unroll
      for (int tt = 0; tt < TP; ++tt) wgmma_fence_operand(acc[tt]);
      wgmma_wait<1>();                           // the previous k-block's MMAs have retired: its stage is free
      if (kb > kb0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[prev]);
      }
      prev = stage;
      if (++stage == C::STAGES) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
#pragma unroll
    for (int tt = 0; tt < TP; ++tt) wgmma_fence_operand(acc[tt]);
    // epilogue: accumulator (row, col) = (output channel, input channel of the tap), column pairs -> float2 atomics
    const long ktot = (long)p.ksize * p.ksize * p.cin;
    const int rbase = co0 + 64 * cw + 16 * (t >> 5) + (lane >> 2);
#pragma unroll
    for (int tt = 0; tt < TP; ++tt) {
#pragma unroll
      for (int i = 0; i < BNW / 2; i += 2) {
        const int co = rbase + 8 * ((i >> 1) & 1);
        const int ci = 8 * (i >> 2) + 2 * (lane & 3);
        if (co < p.cout)
          atomicAdd(reinterpret_cast<float2*>(p.dw + (long)co * ktot + (long)(tap0 + tt) * p.cin + ci0 + ci),
                    make_float2(acc[tt][i], acc[tt][i + 1]));
      }
    }
  }
}

// Stem wgrad (cin = 3): CUDA cores.  Block = 256 output pixels; thread t accumulates the 27 x 32 products of
// its pixel ... reduced per block in shared memory, then atomics.
__global__ void __launch_bounds__(256)
stem_wgrad_kernel(const float* __restrict__ x, const void* __restrict__ dz, int is_bf16, int n, int h, int w,
                  float* __restrict__ dw /*[32][27]*/) {
  __shared__ float s_acc[32 * 27];
  for (int i = threadIdx.x; i < 32 * 27; i += 256) s_acc[i] = 0.f;
  __syncthreads();
  const long P = (long)n * h * w;
  // each warp handles pixels; lane = output channel
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  float acc[27];
#pragma unroll
  for (int k = 0; k < 27; ++k) acc[k] = 0.f;
  for (long pix = (long)blockIdx.x * 8 + wib; pix < P; pix += (long)gridDim.x * 8) {
    const int px = (int)(pix % w), py = (int)((pix / w) % h);
    const long img = pix / ((long)w * h);
    float g;
    if (is_bf16) g = __bfloat162float(static_cast<const __nv_bfloat16*>(dz)[pix * 32 + lane]);
    else g = __half2float(static_cast<const __half*>(dz)[pix * 32 + lane]);
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int s = 0; s < 3; ++s) {
        const int yy = py + r - 1, xx = px + s - 1;
        if (yy >= 0 && yy < h && xx >= 0 && xx < w) {
          const float* xp = x + ((img * h + yy) * w + xx) * 3;
#pragma unroll
          for (int c = 0; c < 3; ++c) acc[(r * 3 + s) * 3 + c] = fmaf(g, __ldg(xp + c), acc[(r * 3 + s) * 3 + c]);
        }
      }
  }
#pragma unroll
  for (int k = 0; k < 27; ++k) atomicAdd(&s_acc[lane * 27 + k], acc[k]);
  __syncthreads();
  for (int i = threadIdx.x; i < 32 * 27; i += 256) atomicAdd(dw + i, s_acc[i]);
}

// Pixel splits (split-K) of one wgrad launch.  One CTA is resident per SM (192 KB of stages), so the grid runs in waves
// of `sms` CTAs, and every CTA ends with TP x BNW x 128 fp32 atomics that nothing overlaps, costed as `epi_blocks` pixel
// blocks' worth of main loop.  Returns the split count that minimises waves x (blocks per CTA + epi).
long wgrad_pick_splits(long num_kb, long tiles, long sms, long epi_blocks) {
  long splits = 1;
  double best = 1e30;
  const long smax = num_kb < 4 * sms ? num_kb : 4 * sms;
  for (long s = 1; s <= smax; ++s) {
    const long kbs = (num_kb + s - 1) / s;
    const long s_eff = (num_kb + kbs - 1) / kbs;
    const long waves = (tiles * s_eff + sms - 1) / sms;
    const double cost = (double)waves * ((double)kbs + (double)epi_blocks);
    if (cost < best - 1e-9) { best = cost; splits = s_eff; }
  }
  return splits;
}

// One conv_wgrad_kernel instantiation: the type wgrad_kernel_for passes to its functor
template <typename T, int BNW, int TP>
struct WgradKernel {
  using C = WCfg<BNW, TP>;
  static constexpr auto kernel = conv_wgrad_kernel<T, BNW, TP>;
};

static int no_wgrad_kernel(const WgradParams& p) {
  set_error("wgrad: no kernel for dtype %d, %d channels per tap, %d taps per CTA", p.dtype, p.bnw, p.tp);
  return YB_ERR_UNSUPPORTED;
}

template <typename T, typename F>
static int wgrad_kernel_type(const WgradParams& p, F& f) {
  if (p.bnw == 128 && p.tp == 1) return f(WgradKernel<T, 128, 1>());
  if (p.bnw == 64 && p.tp == 3) return f(WgradKernel<T, 64, 3>());
  if (p.bnw == 64 && p.tp == 1) return f(WgradKernel<T, 64, 1>());
  if (p.bnw == 32 && p.tp == 3) return f(WgradKernel<T, 32, 3>());
  if (p.bnw == 32 && p.tp == 1) return f(WgradKernel<T, 32, 1>());
  return no_wgrad_kernel(p);
}

// The instantiation table: every conv_wgrad_kernel that exists is named here and nowhere else.  Calls
// f(WgradKernel<...>()) with the instantiation wgrad_select recorded in p and returns what f returns, or
// YB_ERR_UNSUPPORTED when there is none.
template <typename F>
static int wgrad_kernel_for(const WgradParams& p, F&& f) {
  if (p.dtype == YB_F16) return wgrad_kernel_type<__half>(p, f);
  if (p.dtype == YB_BF16) return wgrad_kernel_type<__nv_bfloat16>(p, f);
  return no_wgrad_kernel(p);
}

// Shape checks, kernel and grid of one weight gradient: everything wgrad_prepare decides before it looks at the data
// pointers, down to the conv_wgrad_kernel instantiation, which must exist.
int wgrad_select(const yb_conv_desc* d, int sm_count, WgradParams* p) {
  memset(p, 0, sizeof(*p));
  YB_REQUIRE(d->ksize == 1 || d->ksize == 3, "wgrad: ksize must be 1 or 3");
  YB_REQUIRE(d->stride == 1 || d->stride == 2, "wgrad: stride must be 1 or 2");
  YB_REQUIRE(d->cin > 0 && d->cin % 32 == 0, "wgrad: cin must be a positive multiple of 32 (got %d)", d->cin);
  YB_REQUIRE(d->cout > 0 && d->n > 0 && d->h >= d->stride && d->w >= d->stride, "wgrad: empty problem");
  YB_REQUIRE(d->dtype == YB_F16 || d->dtype == YB_BF16, "wgrad: dtype must be f16 or bf16");
  const int ho = d->h / d->stride, wo = d->w / d->stride;
  const long P = (long)d->n * ho * wo;
  const long num_kb = ceil_div(P, WG_BKP);
  YB_REQUIRE(num_kb <= 0x7fffffff, "wgrad: too many output pixels");
  const int taps = d->ksize * d->ksize;
  // 3x3 convs accumulate one kernel row (3 taps) per CTA, at most 64 input channels per tap: 3 x 64 accumulator columns
  // are 96 registers per thread.  1x1 convs have one tap and take up to 128 channels.
  const int bnw = taps == 1 && d->cin % 128 == 0 ? 128 : (d->cin % 64 == 0 ? 64 : 32);
  const char* tpf = opt("YB_WGRAD_TP");     // "1": one tap per CTA (A/B testing)
  const int tp = (taps == 1 || (tpf && tpf[0] == '1')) ? 1 : 3;
  const int tap_groups = taps / tp;
  const int n_chunks = d->cin / bnw;
  const int co_tiles = ceil_div(d->cout, WG_BM);
  const long tiles = (long)tap_groups * n_chunks * co_tiles;
  long splits;
  if (opt("YB_WGRAD_SPLITS")[0]) {          // forced split count (tests: deep rings, short last splits)
    splits = opt_int("YB_WGRAD_SPLITS", 1);
    splits = splits < 1 ? 1 : (splits > num_kb ? num_kb : splits);
  } else {
    splits = wgrad_pick_splits(num_kb, tiles, sm_count, opt_int("YB_WGRAD_EPI", 40));
  }
  const long kb_per_split = ceil_div(num_kb, splits);
  splits = ceil_div(num_kb, kb_per_split);
  p->P = P; p->ho = ho; p->wo = wo;
  p->cin = d->cin; p->cout = d->cout; p->ksize = d->ksize; p->stride = d->stride; p->pad = d->ksize / 2;
  p->kb_per_split = (int)kb_per_split;
  p->num_kb = (int)num_kb;
  p->n_chunks = n_chunks;
  p->dtype = d->dtype;
  p->bnw = bnw;
  p->tp = tp;
  p->grid_x = (int)splits;
  p->grid_y = tap_groups * n_chunks;
  p->grid_z = co_tiles;
  return wgrad_kernel_for(*p, [](auto) -> int { return YB_OK; });
}

// wgrad_select, then the tensor maps over the data pointers, which are baked into maps and parameters.
int wgrad_prepare(const yb_conv_desc* d, const void* x, const void* dz, int dz_ld, int dz_dilated, float* dw,
                  WgradLaunch* l) {
  YB_REQUIRE(x && dz && dw, "wgrad: null pointer");
  WgradParams* p = &l->p;
  int rc = wgrad_select(d, num_sms(), p);
  if (rc) return rc;
  YB_REQUIRE(dz_ld >= d->cout && dz_ld % 8 == 0 && d->in_ld % 8 == 0, "wgrad: bad leading dimensions");
  p->dw = dw;
  p->a_dilated = dz_dilated ? 1 : 0;
  if (dz_dilated) {
    YB_REQUIRE(d->stride == 2, "wgrad: dz_dilated only applies to stride-2 layers");
    rc = make_tmap_im2col_px(&l->tmA, dz, d->dtype, d->n, d->h, d->w, d->cout, dz_ld, 1, 2, 0, 64, WG_BKP);
  } else {
    rc = make_tmap_2d(&l->tmA, dz, d->dtype, p->P, d->cout, dz_ld, WG_BKP, 64, 0);
  }
  if (rc) return rc;
  return make_tmap_im2col_px(&l->tmB, x, d->dtype, d->n, d->h, d->w, d->cin, d->in_ld, d->ksize, d->stride, p->pad,
                             p->bnw < 64 ? p->bnw : 64, WG_BKP);
}

template <typename K>
static int wgrad_launch_kernel(const WgradLaunch& l, cudaStream_t st) {
  static DeviceOnce once;
  auto kern = K::kernel;
  const int rc = ensure_smem_attr(once, reinterpret_cast<const void*>(kern), K::C::SMEM_BYTES);
  if (rc) return rc;
  const dim3 grid((unsigned)l.p.grid_x, (unsigned)l.p.grid_y, (unsigned)l.p.grid_z);
  kern<<<grid, WG_THREADS, K::C::SMEM_BYTES, st>>>(l.tmA, l.tmB, l.p);
  YB_CUDA(cudaGetLastError());
  return YB_OK;
}

// Launch a prepared weight gradient (wgrad_prepare): the kernel and grid wgrad_select recorded in l.p
int wgrad_launch(const WgradLaunch& l, cudaStream_t st) {
  return wgrad_kernel_for(l.p, [&](auto k) -> int { return wgrad_launch_kernel<decltype(k)>(l, st); });
}

}  // namespace yb

using namespace yb;

// Host-only: the kernel and grid yb_conv2d_wgrad launches for `d` on a device with sm_count SMs, with the current options
// (YB_WGRAD_TP, YB_WGRAD_EPI, YB_WGRAD_SPLITS).
extern "C" int yb_wgrad_schedule(const yb_conv_desc* d, int sm_count, yb_wgrad_schedule_info* info) {
  YB_REQUIRE(d && info && sm_count > 0, "wgrad_schedule: bad argument");
  WgradParams p;
  int rc = wgrad_select(d, sm_count, &p);
  if (rc) return rc;
  info->bnw = p.bnw;
  info->tp = p.tp;
  rc = wgrad_kernel_for(p, [&](auto k) -> int { info->stages = decltype(k)::C::STAGES; return YB_OK; });
  if (rc) return rc;
  info->num_kb = p.num_kb;
  info->kb_per_split = p.kb_per_split;
  info->splits = p.grid_x;
  info->tiles = p.grid_y * p.grid_z;
  info->grid_x = p.grid_x;
  info->grid_y = p.grid_y;
  info->grid_z = p.grid_z;
  return YB_OK;
}

extern "C" int yb_conv2d_wgrad(const yb_conv_desc* d, const void* x, const void* dz, int dz_ld, int dz_dilated,
                               float* dw, void* stream) {
  YB_REQUIRE(d, "wgrad: null pointer");
  WgradLaunch l;
  int rc = wgrad_prepare(d, x, dz, dz_ld, dz_dilated, dw, &l);
  if (rc) return rc;
  return wgrad_launch(l, static_cast<cudaStream_t>(stream));
}

extern "C" int yb_stem_conv_wgrad_tc(const float* x, const void* dz, int dtype, int n, int h, int w, float* dw,
                                     void* stream);
extern "C" int yb_stem_conv_wgrad(const float* x, const void* dz, int dtype, int n, int h, int w, float* dw,
                                  void* stream) {
  YB_REQUIRE(x && dz && dw && n > 0 && h > 0 && w > 0, "stem_wgrad: bad argument");
  YB_REQUIRE(dtype == YB_F16 || dtype == YB_BF16, "stem_wgrad: dtype must be f16 or bf16");
  {
    const char* sw = opt("YB_STEM_WGRAD");   // "cuda": the CUDA-core kernel below (A/B testing)
    if (!(sw && sw[0] == 'c')) return yb_stem_conv_wgrad_tc(x, dz, dtype, n, h, w, dw, stream);
  }
  const long P = (long)n * h * w;
  long blocks = (P + 7) / 8;
  const long cap = (long)num_sms() * 8;
  if (blocks > cap) blocks = cap;
  stem_wgrad_kernel<<<(int)blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(x, dz, dtype == YB_BF16, n, h, w, dw);
  YB_CUDA(cudaGetLastError());
  return YB_OK;
}
