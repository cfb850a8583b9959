// 3x3 convolution for the Cin <= 64 layers at the top of Darknet-53 (utils/layer_utils.py:35-44: Conv_1 32->64 /2,
// Conv_3 32->64, Conv_4 64->128 /2, Conv_6 / Conv_8 64->128) on the tensor cores, with the A operand taken from a
// shared-memory HALO TILE instead of nine im2col gathers.
//
// Why: with 32 / 64 input channels an im2col row is 64 / 128 bytes and one k-block is one filter tap, so the generic
// implicit-GEMM kernel (conv_igemm.cu) issues 9 TMA requests of 128 rows per 128-pixel tile — every input pixel is
// fetched 9x from L2 and the TMA row rate (not bandwidth, not the MMA) paces the layer.  Here:
//   * a tile is 16 x 8 output pixels (M = 128: sixteen 8-row groups, group g = output row g; two consumer warpgroups
//     own output rows 0..7 and 8..15 and issue wgmma m64nCOUTk16);
//   * stride 1: ONE tiled TMA load brings the (16+2) x (8+2) input halo [18][10][Cin] into shared memory (borders and
//     the bottom tail zero-filled by the TMA), 1.4x instead of 9x the tile's pixels;
//     stride 2: four loads with traversal stride 2 bring the four (row, col)-parity planes of the 33 x 17 halo, so
//     that every tap again reads a dense window of one plane;
//   * tap (r, s) needs NO data movement: its A operand is the same shared-memory tile, addressed by a wgmma descriptor
//     that starts (dr * plane_width + ds) rows further down and uses the plane width as the 8-row-group stride (SBO).
//     The 128B / 64B swizzle is a function of the shared-memory address bits, so a descriptor may start at any row of
//     a TMA-written tile;
//   * all 9 taps' weights [Cout][9 * Cin] stay resident in shared memory for the whole persistent CTA;
//   * 16-bit outputs: the TMA-store epilogue of conv_igemm.cu (epi_box_to_slab): each consumer warp applies scale /
//     shift, leaky and the residual to its fragments in registers, writes them by stmatrix into a swizzled slab and
//     stores its 2 output rows x 8 pixels x 64 channels with one 4D TMA store, without a warpgroup barrier.  The
//     e4m3 output and a residual read from global memory (YB_CONV_RES=ldg) keep the staging-tile epilogue, with
//     pixel (not row) addressing.
// Warp roles: warp 0 TMA producer, warps 4..11 (warpgroups 1, 2) MMA + epilogue, fp32 accumulators in registers; the
// producer keeps up to NST halo tiles in flight ahead of the MMAs.
// Inference only (folded BN): scale/shift + leaky + optional residual, 16-bit NHWC in and out.  One instantiation
// (TO = e4m3, fp16 in) writes the first e4m3 buffer of the fp8 plan: Conv_3, whose fp16 residual is read as usual.
#include <cudaTypedefs.h>
#include <string.h>

#include <type_traits>

#include "common.cuh"
#include "conv.cuh"
#include "wgmma.cuh"

namespace yb {

int make_tmap_2d(CUtensorMap* tm, const void* base, int dtype, long rows, long cols, long ld, int box_rows, int box_cols,
                 int weights);
int make_tmap_image3d(CUtensorMap* tm, const float* base, int n, int h, int w, int box_f, int box_h);
int make_tmap_tiled4d(CUtensorMap* tm, const void* base, int dtype, int n, int h, int w, int c, long ld, int box_c,
                      int box_w, int box_h, int estride);

static constexpr int HT_H = 16, HT_W = 8;       // output tile
static constexpr int HALO_THREADS = 384;         // warp 0: TMA, warpgroups 1, 2: MMA + epilogue
static constexpr int HALO_EPI_LD = 33;          // staging row pitch in floats

// Fused stem (darknet53_body/Conv, 3 -> 32, 3x3/1, utils/layer_utils.py:35) as the PRODUCER of Conv_1's parity planes:
// the 709 MB stem output of a batch-64 step is never written nor re-read.  Per 16x8-pixel tile of Conv_1 the stem is
// needed on 33 x 17 pixels; their 35 x 19-pixel float32 input halo arrives by one 3D TMA load, STEMW producer warps
// compute the stem on mma.sync (m16n8k16: A = the 27 -> 32 patch values gathered straight from the halo, B = the stem
// weights held in registers), apply BN + leaky and store the 16-bit results into the swizzled plane tiles the
// wgmma descriptors of Conv_1 read.  Stem pixels outside the image are Conv_1's zero padding (utils/layer_utils.py:15-16).
struct StemCfg {
  static constexpr int SH = 2 * HT_H + 1, SW = 2 * HT_W + 1;             // stem pixels per tile: 33 x 17
  static constexpr int NPX = SH * SW;                                     // 561
  static constexpr int NT16 = (NPX + 15) / 16;                            // 36 m16 tiles
  static constexpr int IN_ROWS = SH + 2;                                  // 35 image rows
  static constexpr int IN_ROWF = 60;                                      // floats per halo row: 19 px x 3 = 57, padded to 16 bytes
  static constexpr int IN_BYTES = (IN_ROWS * IN_ROWF * 4 + 127) / 128 * 128;
  // The planes are written by producer warps of the same CTA, so two stages (one being filled, one being read) keep
  // the consumers fed; the image halo is the layer's only HBM load, so the rest of shared memory goes to its ring.
  // (Measured: 4 plane stages with 3 image stages time the same within 1.5 %; DESIGN.md §5.)
  static constexpr int NST = 2;                                           // plane stages
  static constexpr int NIN_MAX = 8;                                       // image-halo stages
};

// RES (Conv_3: 32 -> 64, stride 1, with a shortcut): every stage also holds the tile's residual, a [16][8] x 64-channel
// box of 128B-swizzled pixel rows loaded by TMA with the halo, so the epilogue adds it from shared memory.
// TMA: the 16-bit outputs' TMA-store epilogue.  Its per-warp output slabs (8 x 2 KB) alias the staging tile, which a
// launch with a global-read residual still uses; with RES the slabs are the stage's residual box itself, and only the
// e4m3 output keeps a staging tile of its own.
// STEMW > 0: the fused stem's plane ring (StemCfg::NST) and image-halo ring (NIN) share the space left by the weights.
template <int CIN, int COUT, int STRIDE, bool RES = false, bool TMA = false, int STEMW = 0>
struct HaloCfg {
  static constexpr int ROWB = CIN * 2;                                   // bytes per pixel row of a plane (one swizzle span)
  static constexpr int NPLANE = STRIDE == 1 ? 1 : 4;
  // plane geometry: stride 1: one [18][10] plane; stride 2: (odd|even rows) x (odd|even cols): 17|16 x 9|8
  static constexpr int ph(int p) { return STRIDE == 1 ? HT_H + 2 : ((p >> 1) == 0 ? HT_H + 1 : HT_H); }
  static constexpr int pw(int p) { return STRIDE == 1 ? HT_W + 2 : ((p & 1) == 0 ? HT_W + 1 : HT_W); }
  static constexpr int pbytes(int p) { return (ph(p) * pw(p) * ROWB + 1023) / 1024 * 1024; }
  static constexpr int poff(int p) { return p == 0 ? 0 : poff(p - 1) + pbytes(p - 1); }
  static constexpr int RES_OFF = poff(NPLANE - 1) + pbytes(NPLANE - 1);  // 1024-byte aligned
  static constexpr int RES_BYTES = RES ? HT_H * HT_W * COUT * 2 : 0;
  static constexpr int STAGE_BYTES = RES_OFF + RES_BYTES;
  static constexpr int STAGE_TX = (STRIDE == 1 ? ph(0) * pw(0) * ROWB
                                               : (ph(0) * pw(0) + ph(1) * pw(1) + ph(2) * pw(2) + ph(3) * pw(3)) * ROWB) +
                                  RES_BYTES;
  static constexpr int B_TAP_BYTES = COUT * ROWB;                        // one tap's [COUT][CIN] weight tile
  static constexpr int B_BYTES = 9 * B_TAP_BYTES;
  // a [64][33] fp32 staging tile per consumer warpgroup, or (TMA) a 16-row x 128-byte output slab per consumer warp
  static constexpr int EPI_BYTES = (TMA && RES) ? 0 : ((TMA && STEMW > 0) ? 8 * 2048 : 2 * 64 * HALO_EPI_LD * 4);
  static constexpr int MISC_BYTES = 1024;                                // barriers
  static constexpr int SS_BYTES = 4 * COUT * 4;                          // scale / shift, per column and per column pair
  static constexpr int BUDGET = 227 * 1024 - 1024 /*alignment slack*/;
  static constexpr int FIXED = B_BYTES + EPI_BYTES + MISC_BYTES + SS_BYTES;
  static constexpr int NST_RAW = (BUDGET - FIXED) / STAGE_BYTES;
  static constexpr int NST = STEMW > 0 ? StemCfg::NST : (NST_RAW > 6 ? 6 : NST_RAW);
  static_assert(NST >= 1 && NST <= 8, "halo conv: configuration does not fit shared memory");
  static constexpr int NIN_RAW = STEMW > 0 ? (BUDGET - FIXED - NST * STAGE_BYTES) / StemCfg::IN_BYTES : 0;
  static constexpr int NIN = NIN_RAW > StemCfg::NIN_MAX ? StemCfg::NIN_MAX : NIN_RAW;   // image-halo stages (STEMW > 0)
  static_assert(STEMW == 0 || NIN >= 2, "halo conv: the fused stem's image ring does not fit shared memory");
  static constexpr int SMEM_BYTES = 1024 + FIXED + NST * STAGE_BYTES + NIN * StemCfg::IN_BYTES;
  static constexpr uint32_t SWIZZLE = ROWB;                              // 128B / 64B: a pixel row is one swizzle span
  // tap (r, s) -> plane and row/col offset inside it.  stride 2 (pad 1 + VALID): input row 2i + r - 1:
  //   r = 0 -> odd-row plane, offset 0; r = 1 -> even-row plane, offset 0; r = 2 -> odd-row plane, offset 1
  static constexpr int tap_plane(int r, int s) { return STRIDE == 1 ? 0 : (((r == 1) ? 2 : 0) | ((s == 1) ? 1 : 0)); }
  static constexpr int tap_dr(int r) { return STRIDE == 1 ? r : (r == 2 ? 1 : 0); }
  static constexpr int tap_ds(int s) { return STRIDE == 1 ? s : (s == 2 ? 1 : 0); }
};

__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void mma16816_f16(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1, bool bf16) {
  if (bf16)
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
  else
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

template <typename T, int CIN, int COUT, int STRIDE, int STEMW = 0, typename TO = T, bool RES = false>
__global__ void __launch_bounds__(HALO_THREADS + 32 * STEMW, 1)
conv_halo_kernel(const __grid_constant__ HaloMaps maps, const __grid_constant__ HaloParams p) {
  constexpr bool kTMA = !std::is_same<TO, __nv_fp8_e4m3>::value;   // 16-bit output: the TMA-store epilogue
  using C = HaloCfg<CIN, COUT, STRIDE, RES, kTMA, STEMW>;
  static_assert(!RES || (CIN == 32 && COUT == 64 && STRIDE == 1 && STEMW == 0), "the residual box is Conv_3's");
  constexpr int PROD_WARP0 = HALO_THREADS / 32;  // first stem-producer warp
  static_assert(STEMW == 0 || (CIN == 32 && STRIDE == 2), "the fused stem feeds Conv_1 (32 -> 64, stride 2)");
  static_assert(STEMW == 0 || kTMA, "the fused stem's Conv_1 has a 16-bit output");
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);   // pointer arithmetic: stays in the shared space
  uint8_t* sB = smem;                                        // [9][COUT][CIN]   swizzled, resident
  uint8_t* sA = smem + C::B_BYTES;                           // [NST][planes]    swizzled halo tiles
  // [2 warpgroups][64][HALO_EPI_LD] staging, or (TMA, not RES) [8 consumer warps][16][128 B] output slabs (1024-byte aligned)
  float* sE = reinterpret_cast<float*>(sA + C::NST * C::STAGE_BYTES);
  uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(sE) + C::EPI_BYTES);
  uint64_t* full_bar = bars;            // [NST]
  uint64_t* empty_bar = bars + 8;       // [NST] one arrive per consumer warp
  uint64_t* b_bar = bars + 20;
  uint64_t* in_full = bars + 32;        // [NIN] float32 input halo landed (TMA -> stem producers)
  uint64_t* in_empty = bars + 48;       // [NIN] stem producers -> TMA
  float* s_ss = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(sE) + C::EPI_BYTES + C::MISC_BYTES);   // [2][COUT] scale / shift
  float* s_ss4 = s_ss + 2 * COUT;       // [COUT / 2] (scale, scale, shift, shift) per column pair: the TMA epilogue's
  uint8_t* sIn = reinterpret_cast<uint8_t*>(s_ss + 4 * COUT);                  // [NIN][35][60] float32 (STEMW > 0 only; 128-byte aligned)

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (warp == 0 && lane == 0) {
    if (STEMW == 0) {                            // (with the fused stem the plane maps are unused and zeroed)
#pragma unroll
      for (int i = 0; i < C::NPLANE; ++i) tma_prefetch_desc(&maps.plane[i]);
    }
    tma_prefetch_desc(&maps.w);
    if (RES) tma_prefetch_desc(&maps.res);
    if (kTMA) tma_prefetch_desc(&maps.out);
    for (int i = 0; i < C::NST; ++i) { mbar_init(&full_bar[i], STEMW > 0 ? STEMW : 1); mbar_init(&empty_bar[i], 8); }
    if (STEMW > 0) {
      tma_prefetch_desc(&maps.in3d);
      for (int i = 0; i < C::NIN; ++i) { mbar_init(&in_full[i], 1); mbar_init(&in_empty[i], STEMW); }
    }
    mbar_init(b_bar, 1);
    fence_barrier_init();
  }
  for (int c = threadIdx.x; c < COUT; c += blockDim.x) {
    const float sc = c < p.cout ? __ldg(p.scale + c) : 0.f, sh = c < p.cout ? __ldg(p.shift + c) : 0.f;
    s_ss[c] = sc;
    s_ss[COUT + c] = sh;
    s_ss4[(c >> 1) * 4 + (c & 1)] = sc;
    s_ss4[(c >> 1) * 4 + 2 + (c & 1)] = sh;
  }
  __syncthreads();

  if (warp == 0) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      mbar_arrive_expect_tx(b_bar, (uint32_t)C::B_BYTES);
#pragma unroll
      for (int t = 0; t < 9; ++t) tma_load_2d(sB + t * C::B_TAP_BYTES, &maps.w, b_bar, t * CIN, 0);
      int stage = 0;
      uint32_t phase = 0;
      if (STEMW > 0) {
        // float32 image halo of the tile: rows 2 h0 - 2 .. 2 h0 + 32, pixels 2 w0 - 2 .. 2 w0 + 16 (x 3 channels),
        // zero-filled outside the image (= the stem's SAME padding)
        for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
          const int tx = tile % p.tiles_x;
          const int ty = (tile / p.tiles_x) % p.tiles_y;
          const int img = tile / (p.tiles_x * p.tiles_y);
          mbar_wait(&in_empty[stage], phase ^ 1);
          mbar_arrive_expect_tx(&in_full[stage], (uint32_t)(StemCfg::IN_ROWS * StemCfg::IN_ROWF * 4));
          // (the innermost TMA coordinate must be 16-byte aligned — an unaligned start is an illegal instruction; the halo's
          //  first float (2 tx 8 - 2) * 3 is always 2 mod 4, so the box starts 2 floats earlier: 2 + 57 <= 60 floats per row)
          tma_load_3d(sIn + stage * StemCfg::IN_BYTES, &maps.in3d, &in_full[stage], (2 * tx * HT_W - 2) * 3 - 2, 2 * ty * HT_H - 2, img);
          if (++stage == C::NIN) { stage = 0; phase ^= 1; }
        }
      }
      for (int tile = blockIdx.x; STEMW == 0 && tile < p.num_tiles; tile += gridDim.x) {
        const int tx = tile % p.tiles_x;
        const int ty = (tile / p.tiles_x) % p.tiles_y;
        const int img = tile / (p.tiles_x * p.tiles_y);
        const int h0 = ty * HT_H, w0 = tx * HT_W;
        mbar_wait(&empty_bar[stage], phase ^ 1);
        mbar_arrive_expect_tx(&full_bar[stage], (uint32_t)C::STAGE_TX);
        uint8_t* dst = sA + stage * C::STAGE_BYTES;
        if (STRIDE == 1) {
          tma_load_4d(dst, &maps.plane[0], &full_bar[stage], 0, w0 - 1, h0 - 1, img);
          if (RES) tma_load_4d(dst + C::RES_OFF, &maps.res, &full_bar[stage], 0, w0, h0, img);   // rows past ho: zeros
        } else {
#pragma unroll
          for (int pl = 0; pl < 4; ++pl) {
            // plane (odd|even rows, odd|even cols): first input row 2 h0 - 1 (odd plane) or 2 h0 (even plane)
            const int hs = 2 * h0 - ((pl >> 1) == 0 ? 1 : 0), ws = 2 * w0 - ((pl & 1) == 0 ? 1 : 0);
            tma_load_4d(dst + C::poff(pl), &maps.plane[pl], &full_bar[stage], 0, ws, hs, img);
          }
        }
        if (++stage == C::NST) { stage = 0; phase ^= 1; }
      }
    }
  } else if (warp >= 4 && warp < PROD_WARP0) {
    // ===================== MMA + epilogue: warpgroup cw owns output rows [8 cw, 8 cw + 8) of every tile =====================
    constexpr bool kBF16 = std::is_same<T, __nv_bfloat16>::value;
    const int cw = (warp - 4) >> 2;
    const int t = threadIdx.x & 127;
    const int bar_id = 1 + cw;
    float* stg = sE + cw * 64 * HALO_EPI_LD;
    const bool has_res = STEMW == 0 && p.res != nullptr;      // (Conv_1 has no shortcut: the residual code is compiled out of the fused kernel)
    const int er = t >> 1, eh = t & 1;                         // epilogue: this thread's pixel of the chunk and its 16-channel half
    const float slope = p.leaky ? 0.1f : 1.f;                  // TMA epilogue: fmaxf(v, 1 v) == v
    const uint32_t a_base = smem_u32(sA), b_base = smem_u32(sB);
    float acc[COUT / 2];
    mbar_wait(b_bar, 0);
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t st_base = a_base + stage * C::STAGE_BYTES;
      wgmma_fence_operand(acc);
      wgmma_fence();
#pragma unroll
      for (int r = 0; r < 3; ++r) {
#pragma unroll
        for (int s = 0; s < 3; ++s) {
          const int pl = C::tap_plane(r, s);
          const uint32_t a_tap = st_base + C::poff(pl) + ((8 * cw + C::tap_dr(r)) * C::pw(pl) + C::tap_ds(s)) * C::ROWB;
          const uint32_t b_tap = b_base + (r * 3 + s) * C::B_TAP_BYTES;
#pragma unroll
          for (int k = 0; k < CIN / 16; ++k)
            Wgmma<COUT, kBF16, 0, 0>::mma(acc, make_kmajor_desc(a_tap + k * 32, C::pw(pl) * C::ROWB, C::SWIZZLE),
                                          make_kmajor_desc(b_tap + k * 32, 8 * C::ROWB, C::SWIZZLE), (r | s | k) != 0);
        }
      }
      wgmma_commit();
      wgmma_fence_operand(acc);
      wgmma_wait<0>();
      wgmma_fence_operand(acc);
      // RES: the stage also holds the residual the epilogue reads, so it is released after the epilogue
      const uint8_t* sres = sA + stage * C::STAGE_BYTES + C::RES_OFF;
      const int rel_stage = stage;
      if (!RES) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[stage]);
      }
      if (++stage == C::NST) { stage = 0; phase ^= 1; }

      const int tx = tile % p.tiles_x;
      const int ty = (tile / p.tiles_x) % p.tiles_y;
      const int img = tile / (p.tiles_x * p.tiles_y);
      if constexpr (kTMA) {
        if (RES || !has_res) {
          // TMA-store epilogue (epi_box_to_slab): warp wq of the warpgroup owns accumulator rows 16 wq .. 16 wq + 15,
          // which are output rows 8 cw + 2 wq and + 1 of the tile, so each 64 channels of them are one {64, 8, 2, 1}
          // box of maps.out (rows at or past ho are clipped by the TMA).  No warpgroup barrier: each warp works alone.
          const int wq = (warp - 4) & 3, oh0 = ty * HT_H + 8 * cw + 2 * wq;
          uint8_t* slab = RES ? sA + rel_stage * C::STAGE_BYTES + C::RES_OFF + (64 * cw + 16 * wq) * 128
                              : reinterpret_cast<uint8_t*>(sE) + (warp - 4) * 2048;
#pragma unroll
          for (int b = 0; b < COUT / 64; ++b) {
            epi_box_to_slab<T, COUT, RES>(acc, b, reinterpret_cast<const float4*>(s_ss4), slab, slope, lane);
            if (lane == 0 && oh0 < p.ho) {
              tma_store_4d(&maps.out, slab, 64 * b, tx * HT_W, oh0, img);
              bulk_commit_group();
            }
          }
          if (RES && lane == 0) {                // the store has read the residual box: the stage may be refilled
            bulk_wait_group_read<0>();
            mbar_arrive(&empty_bar[rel_stage]);
          }
          continue;
        }
      }
      // staged epilogue: the e4m3 output, and a residual read from global memory (YB_CONV_RES=ldg)
      const int oh = ty * HT_H + 8 * cw + (er >> 3), ow = tx * HT_W + (er & 7);
      const bool ok = oh < p.ho && ow < p.wo;
      const long off = ((long)img * p.ho + oh) * p.wo + ow;
#pragma unroll 1
      for (int ch = 0; ch < COUT / 32; ++ch) {
        warpgroup_bar(bar_id);                   // the previous chunk's readers are done with the staging tile
        wgmma_stage_chunk<COUT>(acc, ch, stg, HALO_EPI_LD, t);
        warpgroup_bar(bar_id);
        if (!ok) continue;
        const int c0 = ch * 32 + eh * 16;
        const float* src = stg + er * HALO_EPI_LD + eh * 16;
        float v[16];
#pragma unroll
        for (int j = 0; j < 16; ++j) v[j] = fmaf(src[j], s_ss[c0 + j], s_ss[COUT + c0 + j]);
        if (p.leaky) {
#pragma unroll
          for (int j = 0; j < 16; ++j) v[j] = fmaxf(v[j], 0.1f * v[j]);
        }
        if (has_res) {
          const uint4* rp = reinterpret_cast<const uint4*>(static_cast<const T*>(p.res) + off * p.res_ld + c0);
          // RES: pixel 64 cw + er of the [16][8] box, 16-byte chunks c0 / 8 and c0 / 8 + 1 stored at chunk ^ (pixel & 7)
          const int px = 64 * cw + er;
          const uint8_t* rrow = sres + px * 128;
#pragma unroll
          for (int j = 0; j < 2; ++j) {
            const uint4 u = RES ? *reinterpret_cast<const uint4*>(rrow + ((((c0 >> 3) + j) ^ (px & 7)) << 4)) : __ldg(rp + j);
            float2 f;
            f = Pack2<T>::unpack(u.x); v[8 * j + 0] += f.x; v[8 * j + 1] += f.y;
            f = Pack2<T>::unpack(u.y); v[8 * j + 2] += f.x; v[8 * j + 3] += f.y;
            f = Pack2<T>::unpack(u.z); v[8 * j + 4] += f.x; v[8 * j + 5] += f.y;
            f = Pack2<T>::unpack(u.w); v[8 * j + 6] += f.x; v[8 * j + 7] += f.y;
          }
        }
        if constexpr (std::is_same<TO, __nv_fp8_e4m3>::value) {
          *reinterpret_cast<uint4*>(static_cast<uint8_t*>(p.out) + off * p.out_ld + c0) = e4m3x16_pack(v, p.out_inv_scale);
          continue;
        }
        uint4* op = reinterpret_cast<uint4*>(static_cast<T*>(p.out) + off * p.out_ld + c0);
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          uint4 pk;
          pk.x = Pack2<T>::pack(v[8 * j + 0], v[8 * j + 1]);
          pk.y = Pack2<T>::pack(v[8 * j + 2], v[8 * j + 3]);
          pk.z = Pack2<T>::pack(v[8 * j + 4], v[8 * j + 5]);
          pk.w = Pack2<T>::pack(v[8 * j + 6], v[8 * j + 7]);
          op[j] = pk;
        }
      }
      if (RES) {                                 // this warp's last read of the stage is done
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[rel_stage]);
      }
    }
    if constexpr (kTMA) {
      if (lane == 0) bulk_wait_group<0>();       // this warp's output stores are complete before the CTA may exit
    }
  } else if (STEMW > 0 && warp >= PROD_WARP0) {
    // ===================== stem producers (warps PROD_WARP0 .. PROD_WARP0 + STEMW - 1) =====================
    const int pw_id = warp - PROD_WARP0;
    const bool bf16 = std::is_same<T, __nv_bfloat16>::value;
    const int g = lane >> 2, q = lane & 3;         // mma fragment coordinates: row group, column quad
    // B fragments: stem weights W[n][k] (k = (r*3+s)*3+c < 27), n8 tile nt, k-step ks: b0 = k 2q..2q+1, b1 = k + 8
    uint32_t bfrag[4][2][2];
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
#pragma unroll
      for (int ks = 0; ks < 2; ++ks)
#pragma unroll
        for (int hb = 0; hb < 2; ++hb) {
          const int n = nt * 8 + g, k = ks * 16 + hb * 8 + 2 * q;
          const float w0 = k < 27 ? __ldg(p.stem_w + n * 27 + k) : 0.f;
          const float w1 = k + 1 < 27 ? __ldg(p.stem_w + n * 27 + k + 1) : 0.f;
          bfrag[nt][ks][hb] = Pack2<T>::pack(w0, w1);
        }
    float sc[4][2], sh[4][2];
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        sc[nt][j] = __ldg(p.stem_scale + nt * 8 + 2 * q + j);
        sh[nt][j] = __ldg(p.stem_shift + nt * 8 + 2 * q + j);
      }
    // halo offsets of this thread's 8 patch elements: k -> row k / 9, float k % 9 of the 3 x 9 patch
    int koff[2][2][2];
#pragma unroll
    for (int ks = 0; ks < 2; ++ks)
#pragma unroll
      for (int hb = 0; hb < 2; ++hb)
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const int k = ks * 16 + hb * 8 + 2 * q + j;
          koff[ks][hb][j] = k < 27 ? (k / 9) * StemCfg::IN_ROWF + (k % 9) : 0;
        }
    int in_stage = 0, stage = 0;
    uint32_t in_phase = 0, phase = 0;
    for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
      const int tx = tile % p.tiles_x;
      const int ty = (tile / p.tiles_x) % p.tiles_y;
      const int gy0 = 2 * ty * HT_H - 1, gx0 = 2 * tx * HT_W - 1;      // image coordinates of stem pixel (0, 0) of the tile
      mbar_wait(&in_full[in_stage], in_phase);
      mbar_wait(&empty_bar[stage], phase ^ 1);
      const float* halo = reinterpret_cast<const float*>(sIn + in_stage * StemCfg::IN_BYTES) + 2;   // see the TMA coordinate
      uint8_t* planes = sA + stage * C::STAGE_BYTES;
      // The 561 stem pixels are walked PLANE BY PLANE in m16 tiles (10 + 9 + 9 + 8 = 36): a tile lies inside one plane, so
      // the plane's constants are warp-uniform, consecutive fragment rows are consecutive 64-byte rows of the plane tile,
      // and the pixel -> (row, col) split is one constant division (the first version split every pixel index by 17 and
      // selected the plane per pixel: ~250 instructions per m16 tile, issue-bound at 6.5 k cycles per output tile).
      struct M16 {                                 // one m16 tile of stem pixels in flight
        uint32_t a[2][4];
        float acc[4][4];
        int rho[2], poff;
        bool live[2], inside[2];
      };
      auto gather = [&](const int t, M16& m) {
        const int pl = t < 10 ? 0 : (t < 19 ? 1 : (t < 28 ? 2 : 3));              // warp-uniform
        const int t0 = pl == 0 ? 0 : (pl == 1 ? 10 : (pl == 2 ? 19 : 28));
        const int pwid = (pl & 1) == 0 ? HT_W + 1 : HT_W;
        const int npl = ((pl >> 1) == 0 ? HT_H + 1 : HT_H) * pwid;                // pixels of this plane
        m.poff = pl == 0 ? C::poff(0) : (pl == 1 ? C::poff(1) : (pl == 2 ? C::poff(2) : C::poff(3)));
        const int ya = pl >> 1, xb = pl & 1;                                       // stem row = 2 * plane row + ya, col likewise
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {                       // fragment rows g and g + 8
          m.rho[hr] = (t - t0) * 16 + g + 8 * hr;
          m.live[hr] = m.rho[hr] < npl;
          const int r_ = m.live[hr] ? m.rho[hr] : 0;
          const int pr = (pl & 1) == 0 ? r_ / (HT_W + 1) : r_ >> 3;
          const int pc = r_ - pr * pwid;
          const int sy = 2 * pr + ya, sx = 2 * pc + xb;
          m.inside[hr] = m.live[hr] && gy0 + sy >= 0 && gy0 + sy < p.in_h && gx0 + sx >= 0 && gx0 + sx < p.in_w;
          const float* base = halo + sy * StemCfg::IN_ROWF + sx * 3;
#pragma unroll
          for (int ks = 0; ks < 2; ++ks)
#pragma unroll
            for (int hb = 0; hb < 2; ++hb) {
              const float v0 = base[koff[ks][hb][0]];            // (k >= 27: offset 0, a finite value times a zero weight)
              const float v1 = base[koff[ks][hb][1]];
              m.a[ks][hb * 2 + hr] = Pack2<T>::pack(v0, v1);     // a0: row g, k lo; a1: row g+8, k lo; a2: row g, k hi; a3: row g+8, k hi
            }
        }
      };
      auto multiply = [&](M16& m) {
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
          m.acc[nt][0] = m.acc[nt][1] = m.acc[nt][2] = m.acc[nt][3] = 0.f;
#pragma unroll
          for (int ks = 0; ks < 2; ++ks) mma16816_f16(m.acc[nt], m.a[ks], bfrag[nt][ks][0], bfrag[nt][ks][1], bf16);
        }
      };
      auto store = [&](const M16& m) {
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
          if (!m.live[hr]) continue;
          uint8_t* row = planes + m.poff + m.rho[hr] * 64 + q * 4;
          const int swz = (m.rho[hr] >> 1) & 3;
          if (m.inside[hr]) {
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) {
              float v0 = fmaf(m.acc[nt][2 * hr], sc[nt][0], sh[nt][0]);
              float v1 = fmaf(m.acc[nt][2 * hr + 1], sc[nt][1], sh[nt][1]);
              v0 = fmaxf(v0, 0.1f * v0); v1 = fmaxf(v1, 0.1f * v1);      // leaky_relu(0.1), model.py:47
              *reinterpret_cast<uint32_t*>(row + ((nt ^ swz) << 4)) = Pack2<T>::pack(v0, v1);
            }
          } else {                                                        // outside the image: Conv_1's zero padding
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) *reinterpret_cast<uint32_t*>(row + ((nt ^ swz) << 4)) = 0u;
          }
        }
      };
      // The 561 stem pixels are walked PLANE BY PLANE in m16 tiles (10 + 9 + 9 + 8 = 36): a tile lies inside one plane, so
      // the plane's constants are warp-uniform and consecutive fragment rows are consecutive 64-byte rows of the plane tile.
      // The producers are latency-bound, not issue-bound: 12 warps (3 m16 tiles each) beat 8 (4 or 5 tiles) and 9 (4
      // tiles); keeping TWO tiles in flight per warp lost to the register pressure and was dropped (DESIGN.md §5).
#pragma unroll 1
      for (int t = pw_id; t < StemCfg::NT16; t += STEMW) {
        M16 m0;
        gather(t, m0);
        multiply(m0);
        store(m0);
      }
      fence_proxy_async();                       // generic-proxy plane writes -> visible to wgmma (async proxy)
      __syncwarp();
      if (lane == 0) {
        mbar_arrive(&full_bar[stage]);
        mbar_arrive(&in_empty[in_stage]);
      }
      if (++in_stage == C::NIN) { in_stage = 0; in_phase ^= 1; }
      if (++stage == C::NST) { stage = 0; phase ^= 1; }
    }
  }
}

static constexpr int STEM_WARPS = 12;          // stem producer warps of the fused kernel (768 threads per CTA)

// One conv_halo_kernel instantiation: the type halo_kernel_for passes to its functor
template <typename T, int CIN, int COUT, int STRIDE, int STEMW = 0, typename TO = T, bool RES = false>
struct HaloKernel {
  static constexpr int THREADS = HALO_THREADS + 32 * STEMW;
  static constexpr int SMEM_BYTES =
      HaloCfg<CIN, COUT, STRIDE, RES, !std::is_same<TO, __nv_fp8_e4m3>::value, STEMW>::SMEM_BYTES;
  static_assert(SMEM_BYTES <= 227 * 1024, "halo conv: configuration does not fit shared memory");
  static constexpr auto kernel = conv_halo_kernel<T, CIN, COUT, STRIDE, STEMW, TO, RES>;
};

static int no_halo_kernel(const HaloParams& p) {
  set_error("conv_halo: no kernel for dtype %d, cin=%d cout=%d stride=%d, fused stem %d, e4m3 output %d, residual box %d",
            p.dtype, p.cin, p.cout, p.stride, p.stem, p.out_e4m3, p.res_smem);
  return YB_ERR_UNSUPPORTED;
}

template <typename T, typename F>
static int halo_kernel_type(const HaloParams& p, F& f) {
  const int ci = p.cin, co = p.cout, s = p.stride;
  if (p.stem) {
    if (ci == 32 && co == 64 && s == 2 && !p.out_e4m3 && !p.res_smem) return f(HaloKernel<T, 32, 64, 2, STEM_WARPS>());
    return no_halo_kernel(p);
  }
  if (ci == 32 && co == 64 && s == 1) {   // Conv_3: the residual box, and (fp16 in) the fp8 plan's e4m3 output
    if (!p.out_e4m3) return p.res_smem ? f(HaloKernel<T, 32, 64, 1, 0, T, true>()) : f(HaloKernel<T, 32, 64, 1>());
    if constexpr (std::is_same<T, __half>::value)
      return p.res_smem ? f(HaloKernel<T, 32, 64, 1, 0, __nv_fp8_e4m3, true>()) : f(HaloKernel<T, 32, 64, 1, 0, __nv_fp8_e4m3>());
    return no_halo_kernel(p);
  }
  if (p.out_e4m3 || p.res_smem) return no_halo_kernel(p);
  if (ci == 32 && co == 64 && s == 2) return f(HaloKernel<T, 32, 64, 2>());
  if (ci == 32 && co == 128 && s == 1) return f(HaloKernel<T, 32, 128, 1>());
  if (ci == 32 && co == 128 && s == 2) return f(HaloKernel<T, 32, 128, 2>());
  if (ci == 64 && co == 64 && s == 1) return f(HaloKernel<T, 64, 64, 1>());
  if (ci == 64 && co == 64 && s == 2) return f(HaloKernel<T, 64, 64, 2>());
  if (ci == 64 && co == 128 && s == 1) return f(HaloKernel<T, 64, 128, 1>());
  return no_halo_kernel(p);   // (64 -> 128 at stride 2: the weights and one parity-plane stage exceed shared memory)
}

// The instantiation table: every conv_halo_kernel that exists is named here and nowhere else.  Calls
// f(HaloKernel<...>()) with the instantiation halo_select recorded in p and returns what f returns, or
// YB_ERR_UNSUPPORTED when there is none.
template <typename F>
static int halo_kernel_for(const HaloParams& p, F&& f) {
  if (p.dtype == YB_F16) return halo_kernel_type<__half>(p, f);
  if (p.dtype == YB_BF16) return halo_kernel_type<__nv_bfloat16>(p, f);
  return no_halo_kernel(p);
}

template <typename K>
static int halo_launch_kernel(const HaloLaunch& l, cudaStream_t st) {
  static DeviceOnce once;
  auto kern = K::kernel;
  const int rc = ensure_smem_attr(once, reinterpret_cast<const void*>(kern), K::SMEM_BYTES);
  if (rc) return rc;
  const int grid = l.p.num_tiles < num_sms() ? l.p.num_tiles : num_sms();
  kern<<<grid, K::THREADS, K::SMEM_BYTES, st>>>(l.maps, l.p);
  YB_CUDA(cudaGetLastError());
  return YB_OK;
}

// Launch a prepared halo-tile conv (conv_halo_prepare): the kernel halo_select recorded in l.p, with the maps built for it
int conv_halo_launch(const HaloLaunch& l, cudaStream_t st) {
  return halo_kernel_for(l.p, [&](auto k) -> int { return halo_launch_kernel<decltype(k)>(l, st); });
}

// Shape checks, tiling and kernel of one halo-tile conv: everything conv_halo_prepare decides before it looks at the
// data pointers, down to the conv_halo_kernel instantiation, which must exist.  The launches, conv_halo_supported and
// yb_net_layer_schedule all select through here.
int halo_select(const HaloRequest& r, HaloParams* p) {
  memset(p, 0, sizeof(*p));
  const yb_conv_desc* d = &r.d;
  YB_REQUIRE(d->ksize == 3 && (d->stride == 1 || d->stride == 2), "conv_halo: 3x3 stride 1|2 only (got k=%d s=%d)",
             d->ksize, d->stride);
  YB_REQUIRE(!d->out_fp32 && !d->upsample2x, "conv_halo: 16-bit, non-upsampled outputs only");
  YB_REQUIRE(d->h % d->stride == 0 && d->w % d->stride == 0 && (d->w / d->stride) % HT_W == 0,
             "conv_halo: h, w must be multiples of the stride and the output width of %d (got %d x %d)", HT_W, d->h, d->w);
  YB_REQUIRE(d->out_ld >= d->cout && d->out_ld % 8 == 0, "conv_halo: out_ld %d invalid", d->out_ld);
  if (r.stem) {
    YB_REQUIRE(!r.res && !r.out_e4m3, "conv_halo: the fused stem's Conv_1 has no residual and a 16-bit output");
  } else {
    YB_REQUIRE(d->in_ld >= d->cin && d->in_ld % 8 == 0, "conv_halo: in_ld %d invalid", d->in_ld);
  }
  // e4m3 codes are stored 16 channels (16 bytes) at a time
  if (r.out_e4m3) YB_REQUIRE(d->out_ld % 16 == 0, "conv_halo: an e4m3 output needs out_ld %% 16 == 0 (got %d)", d->out_ld);
  if (r.res) YB_REQUIRE(d->res_ld >= d->cout && d->res_ld % 8 == 0, "conv_halo: res_ld %d invalid", d->res_ld);
  p->n = d->n; p->ho = d->h / d->stride; p->wo = d->w / d->stride;
  p->tiles_x = p->wo / HT_W; p->tiles_y = ceil_div(p->ho, HT_H);
  p->num_tiles = p->tiles_x * p->tiles_y * d->n;
  p->cout = d->cout; p->leaky = d->leaky;
  p->res_ld = d->res_ld; p->out_ld = d->out_ld;
  if (r.stem) { p->in_h = d->h; p->in_w = d->w; }
  p->out_e4m3 = r.out_e4m3;
  // the residual of Conv_3's shape is TMA-loaded with the halo unless YB_CONV_RES=ldg
  p->res_smem = (r.res && !r.stem && d->cin == 32 && d->cout == 64 && d->stride == 1 &&
                 strcmp(opt("YB_CONV_RES"), "ldg") != 0) ? 1 : 0;
  p->dtype = d->dtype; p->cin = d->cin; p->stride = d->stride; p->stem = r.stem;
  return halo_kernel_for(*p, [](auto) -> int { return YB_OK; });
}

bool conv_halo_supported(const yb_conv_desc* d) {
  HaloParams p;
  return halo_select(HaloRequest{*d}, &p) == YB_OK;
}

// halo_select, then the tensor maps over the data pointers, which are baked into maps and parameters.
int conv_halo_prepare(const HaloRequest& r, const void* x, const void* w_packed, const float* scale, const float* shift,
                      const void* res, void* out, const float* stem_w, const float* stem_scale, const float* stem_shift,
                      HaloLaunch* l) {
  HaloParams* p = &l->p;
  HaloMaps* maps = &l->maps;
  int rc = halo_select(r, p);
  if (rc) return rc;
  const yb_conv_desc* d = &r.d;
  YB_REQUIRE(x && w_packed && scale && shift && out, "conv_halo: null pointer");
  YB_REQUIRE(r.stem ? stem_w && stem_scale && stem_shift : !stem_w && !stem_scale && !stem_shift,
             "conv_halo: the stem's weights, scale and shift are given exactly when the request fuses the stem");
  YB_REQUIRE((res != nullptr) == r.res, "conv_halo: a residual pointer is given exactly when the request has a residual");
  YB_REQUIRE(((uintptr_t)x & 15) == 0 && ((uintptr_t)w_packed & 15) == 0 && ((uintptr_t)out & 15) == 0 && ((uintptr_t)res & 15) == 0,
             "conv_halo: pointers must be 16-byte aligned");
  memset(maps, 0, sizeof(*maps));
  p->scale = scale; p->shift = shift; p->res = res; p->out = out;
  p->stem_w = stem_w; p->stem_scale = stem_scale; p->stem_shift = stem_shift;
  if (p->res_smem) {
    // the residual as {C, W, H, N} = [n, ho, wo, res_ld]: one 64-channel x 8 x 16-pixel box per tile
    rc = make_tmap_tiled4d(&maps->res, res, d->dtype, d->n, p->ho, p->wo, d->cout, d->res_ld, 64, HT_W, HT_H, 1);
    if (rc) return rc;
  }
  if (!p->out_e4m3) {
    // the output as {C, W, H, N}: a consumer warp's 16 accumulator rows are 2 output rows of 8 pixels
    rc = make_tmap_tiled4d(&maps->out, out, d->dtype, d->n, p->ho, p->wo, d->cout, d->out_ld, 64, HT_W, 2, 1);
    if (rc) return rc;
  }
  if (r.stem) {
    // the image's float32 halo of a tile (the plane maps stay zeroed: the stem producers write the planes)
    rc = make_tmap_image3d(&maps->in3d, static_cast<const float*>(x), d->n, d->h, d->w, StemCfg::IN_ROWF, StemCfg::IN_ROWS);
    if (rc) return rc;
  } else if (d->stride == 1) {
    rc = make_tmap_tiled4d(&maps->plane[0], x, d->dtype, d->n, d->h, d->w, d->cin, d->in_ld, d->cin, HT_W + 2, HT_H + 2, 1);
    if (rc) return rc;
  } else {
    for (int pl = 0; pl < 4; ++pl) {
      // traversal stride 2: a box spanning 2 * count - 1 elements loads `count` of them
      const int rows = (pl >> 1) == 0 ? HT_H + 1 : HT_H, cols = (pl & 1) == 0 ? HT_W + 1 : HT_W;
      rc = make_tmap_tiled4d(&maps->plane[pl], x, d->dtype, d->n, d->h, d->w, d->cin, d->in_ld, d->cin, 2 * cols - 1,
                             2 * rows - 1, 2);
      if (rc) return rc;
    }
  }
  const long K = 9L * d->cin;
  return make_tmap_2d(&maps->w, w_packed, d->dtype, yb_conv_cout_pad(d->cout), K, K, d->cout, d->cin, 1);
}

}  // namespace yb

using namespace yb;

extern "C" int yb_conv3x3_halo_supported(const yb_conv_desc* d) { return d && conv_halo_supported(d) ? 1 : 0; }

extern "C" int yb_conv3x3_halo_fwd(const yb_conv_desc* d, const void* x, const void* w_packed, const float* scale,
                                   const float* shift, const void* res, void* out, void* stream) {
  if (!d) { set_error("conv_halo: null descriptor"); return YB_ERR_INVALID_ARGUMENT; }
  HaloRequest r{*d};
  r.res = res != nullptr;
  HaloLaunch l;
  int rc = conv_halo_prepare(r, x, w_packed, scale, shift, res, out, nullptr, nullptr, nullptr, &l);
  if (rc) return rc;
  return conv_halo_launch(l, static_cast<cudaStream_t>(stream));
}

// Stem + Conv_1 in one kernel (utils/layer_utils.py:35-36): image float32 [n, h, w, 3] -> Conv_1's output [n, h/2, w/2, out_ld].
// d describes Conv_1 (h, w = image size = the stem's output size).  The stem's BN is folded into stem_scale / stem_shift.
extern "C" int yb_stem_conv1_fused_fwd(const yb_conv_desc* d, const float* image, const float* stem_w_ohwi,
                                       const float* stem_scale, const float* stem_shift, const void* w_packed,
                                       const float* scale, const float* shift, void* out, void* stream) {
  if (!d) { set_error("stem_conv1_fused: null descriptor"); return YB_ERR_INVALID_ARGUMENT; }
  HaloRequest r{*d};
  r.stem = true;
  HaloLaunch l;
  int rc = conv_halo_prepare(r, image, w_packed, scale, shift, nullptr, out, stem_w_ohwi, stem_scale, stem_shift, &l);
  if (rc) return rc;
  return conv_halo_launch(l, static_cast<cudaStream_t>(stream));
}
