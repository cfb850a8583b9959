// Fused conv (+BN scale/shift +leaky +residual +2x-upsample +concat-slice store) as an
// im2col-free implicit GEMM on the Hopper tensor cores (wgmma):
//
//   D[M = n*ho*wo pixels, N = cout] = A[M, K = k*k*cin] * B[N, K]^T
//
//   A  : NHWC activations.  3x3 convs: TMA *im2col mode* (cuTensorMapEncodeIm2col) gathers
//        128 consecutive output pixels x 64 channels of one filter tap per request — image
//        borders (the darknet pad-1 rule, utils/layer_utils.py:10-21) and the batch tail
//        come back zero-filled, so no padded copy of the input ever exists (K4 in SURVEY §2.3).
//        1x1 convs: plain 2D tiled TMA over the [M, in_ld] matrix.
//   B  : weights packed OHWI = [cout_pad, k*k*cin] K-major, 2D tiled TMA.
//   D  : fp32 accumulators in registers, wgmma.mma_async m64nBNk16 with both operands read from 128B / 64B-swizzled
//        shared memory.
//   e4m3 (the calibrated fp8 inference plan): the same kernel with 1-byte operands and wgmma m64nBNk32.  The shared-memory
//        layout is byte for byte the fp16 one: a 128-byte k-block row holds 128 channels instead of 64, one k32 step
//        advances the descriptors by 32 bytes like one k16 step, and a tile has half the k-blocks.  The epilogue adds
//        the residual times its buffer's scale and stores RN-satfinite e4m3 codes of value / s_out (ConvParams).
//
// Warp roles (384 threads, persistent over tiles): warpgroup 0 = TMA producer (one thread), warpgroups 1 and 2 =
// MMA + epilogue.  The producer runs ahead through the operand ring in work-unit order.  Two schedules:
//   ping-pong (the default): each consumer warpgroup owns whole 128 x BN tiles (two m64 wgmmas per k16 step) and the
//     two take alternate work units.  A pair of named barriers hands the tensor cores from one warpgroup's main loop
//     to the other's, so one warpgroup's epilogue runs while the other's MMAs run.
//   cooperative (fused-decode detection heads, 1x1 convs with 128-column tiles, YB_CONV_MODE clusters, 1-warpgroup
//     CTAs, register epilogue; conv_select chooses): the NC consumer warpgroups split
//     every tile by rows (64 each), run the k-loop in lockstep and then the epilogue together.
// The epilogue stages 32-column chunks of one 64-row accumulator block through shared memory so that each thread then
// owns 16 consecutive channels of one pixel (two 16-byte stores per output row).  Ping-pong launches with a residual
// (RES) find it already in shared memory: a second producer thread TMA-loads each unit's shortcut tile while the unit's
// main loop runs.  The forward layers of the 16-bit inference plans with a plain 16-bit output skip the staging tile
// (TMA, epilogue_tma): each warp packs its fragments in registers and stores swizzled 16-row slabs by TMA.
//
// Replaces: slim.conv2d/batch_norm/leaky_relu (utils/layer_utils.py:20, model.py:43-49),
// tf.add (utils/layer_utils.py:30), tf.pad (:15-16), resize_nearest_neighbor (:86),
// tf.concat (model.py:62,72).
#include <cudaTypedefs.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <type_traits>

#include "common.cuh"
#include "conv.cuh"
#include "wgmma.cuh"

namespace yb {

static constexpr int WG_ROWS = 64;                // accumulator rows per consumer warpgroup
static constexpr int RING_BYTES = 196 * 1024;     // operand ring (the rest of the 227 KB: staging, scale / shift, stats)
static constexpr int EPI_LD = 33;                 // staging row pitch in floats: row walks and column walks are conflict-free
static constexpr int EPI_FLOATS = WG_ROWS * EPI_LD;

// NC consumer warpgroups per CTA (tile = 64 NC rows x BN); warpgroup 0 is the TMA producer.  Both schedules use the
// same 128-row tile for NC = 2, so they share the ring and the tensor maps.
// BKB = bytes of one k-block row (128 or 64): 64 / 32 channels of fp16 / bf16, 128 / 64 channels of e4m3.
// RES (ping-pong, 16-bit): every consumer warpgroup owns a BLOCK_M x BN shortcut tile in shared memory, TMA-loaded in
// 64-column boxes of 128-byte swizzled rows; the operand ring takes what is left of the 227 KB.
template <int BN, int BKB, int NC, bool RES = false>
struct Cfg {
  static constexpr int BLOCK_M = WG_ROWS * NC;
  static constexpr int THREADS = 128 * (NC + 1);
  static constexpr int A_BYTES = BLOCK_M * BKB;
  static constexpr int B_BYTES = BN * BKB;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int RES_BOX_COLS = 64;                      // 16-bit channels per 128-byte swizzled row
  static constexpr int RES_BOX_BYTES = BLOCK_M * 128;          // one 64-column box of the tile
  static constexpr int RES_TILE_BYTES = BLOCK_M * BN * 2;      // one warpgroup's shortcut tile
  static constexpr int RES_BYTES = RES ? NC * RES_TILE_BYTES : 0;
  static constexpr int FIXED_BYTES = 1024 + NC * EPI_FLOATS * 4 + NC * 4 * BN * 4 + 256;
  static constexpr int RING = RES ? 227 * 1024 - FIXED_BYTES - RES_BYTES : RING_BYTES;
  static constexpr int STAGES = (RING / STAGE_BYTES) > 8 ? 8 : (RING / STAGE_BYTES);
  // ring | [RES: NC x shortcut tile] | NC x staging tile | NC x [2][BN] statistics | NC x [2][BN] scale / shift |
  // barriers.  A ping-pong warpgroup stages its 128-row tile one 64-row half after the other through its own 64-row
  // staging tile, so the budget is the same for both schedules (BN = 128, BKB = 128: 6 x 32 KB ring + 2 x 8.4 KB
  // staging + 4 KB = 214 KB; with RES, 4 x 32 KB ring + 2 x 32 KB shortcut tiles + the same 21 KB = 213 KB).
  static constexpr int SMEM_BYTES = FIXED_BYTES + STAGES * STAGE_BYTES + RES_BYTES;
  static constexpr uint32_t SWIZZLE = BKB;        // a k-block row is exactly one swizzle span (128B / 64B)
  static constexpr uint32_t SBO = 8 * BKB;        // bytes between 8-row groups
};
static_assert(Cfg<256, 128, 2>::SMEM_BYTES <= 227 * 1024, "conv: the widest tile does not fit shared memory");
static_assert(2 * 4 * 16 * 128 <= 2 * EPI_FLOATS * 4, "conv: the warps' 16-row output slabs do not fit the staging tiles");
static_assert(Cfg<128, 128, 2, true>::SMEM_BYTES <= 227 * 1024 && Cfg<128, 128, 2, true>::STAGES >= 4,
              "conv: the shortcut tiles leave too short an operand ring");

// the wgmma of an operand type: m64nBNk16 for fp16 / bf16, m64nBNk32 for e4m3 (both 32 bytes of K per instruction)
template <typename T, int BN>
struct ConvMma { using type = Wgmma<BN, std::is_same<T, __nv_bfloat16>::value, 0, 0>; };
template <int BN>
struct ConvMma<__nv_fp8_e4m3, BN> { using type = WgmmaE4M3<BN>; };

// Work unit -> (m tile, n tile) of this CTA.  A cluster of CM x CN CTAs (CM = 0: p.cluster x 1, the shape read at run
// time) takes a unit of CM consecutive m-tiles x CN consecutive n-tiles, and rank r = rm * CN + rn takes m-tile rm and
// n-tile rn of it.  The host takes CN = 2 only where the n-tile count is even; ranks past the last m-tile still take
// part in the multicasts, their rows all masked.  Inference walks n fastest (the A tiles stay hot in L2 across their
// n tiles); with BN statistics on, m runs fastest so a CTA's tiles share their n tile and its per-CTA column sums are
// flushed to global at most num_n_tiles times.
template <int CM, int CN>
__device__ __forceinline__ int num_units(const ConvParams& p) {
  const int cm = CM ? CM : p.cluster;
  return (p.num_m_tiles + cm - 1) / cm * (p.num_n_tiles / CN);
}
template <int CM, int CN>
__device__ __forceinline__ void unit_coords(const ConvParams& p, int unit, uint32_t rank, int& m_idx, int& n_idx) {
  const int cm = CM ? CM : p.cluster;
  const int m_groups = (p.num_m_tiles + cm - 1) / cm, n_groups = p.num_n_tiles / CN;
  int mg, ng;
  if (p.stat_sum != nullptr) { ng = unit / m_groups; mg = unit - ng * m_groups; }
  else { mg = unit / n_groups; ng = unit - mg * n_groups; }
  m_idx = mg * cm + (int)rank / CN;
  n_idx = ng * CN + (int)rank % CN;
}

// executed by the 128 threads of one consumer warpgroup: add the per-CTA column sums into the global statistics
template <int BN>
__device__ __forceinline__ void stat_flush(const ConvParams& p, float* s_stat, int n0, int t, int bar_id) {
  warpgroup_bar(bar_id);
  for (int c = t; c < BN; c += 128) {
    if (n0 + c < p.cout) {
      atomicAdd(p.stat_sum + n0 + c, s_stat[c]);
      atomicAdd(p.stat_sqsum + n0 + c, s_stat[BN + c]);
    }
    s_stat[c] = 0.f;
    s_stat[BN + c] = 0.f;
  }
  warpgroup_bar(bar_id);
}

// 16 consecutive channels of one accumulator row: scale/shift (+leaky) (+residual) -> 16-bit / fp32 global stores
// (channel-slice, 2x-upsample and parity-scatter aware).  SRES: the residual's two 16-byte halves are read from the
// shared-memory shortcut tile at sr0 / sr1 instead of from global memory (same arithmetic, same result).
template <typename T, bool SRES = false>
__device__ __forceinline__ void epi_store16(const ConvParams& p, const float* src, const int row, const int col0,
                                            const float* sc, const float* sh, const uint4* sr0 = nullptr,
                                            const uint4* sr1 = nullptr) {
  float v[16];
#pragma unroll
  for (int j = 0; j < 16; ++j) v[j] = fmaf(src[j], sc[j], sh[j]);
  if (p.leaky) {
#pragma unroll
    for (int j = 0; j < 16; ++j) v[j] = fmaxf(v[j], 0.1f * v[j]);   // == v > 0 ? v : 0.1 v
  }
  // output row of copy rep (2x upsample: 4 copies): orow0 + (rep >> 1) * W2 + (rep & 1), computed per copy so that no
  // row array is live beside a ping-pong warpgroup's 128 accumulators
  long orow0 = row, W2 = 0;
  int nrep = 1;
  if (p.upsample || p.scatter) {
    const int q = row % p.Q;
    const int pp = (row / p.Q) % p.P;
    const int img = row / (p.Q * p.P);
    const long w2 = 2L * p.Q;
    const long base = ((long)img * 2 * p.P + 2 * pp) * w2 + 2 * q;
    if (p.scatter) {
      orow0 = base + ((p.scatter - 1) >> 1) * w2 + ((p.scatter - 1) & 1);
    } else {
      orow0 = base; W2 = w2;
      nrep = 4;
    }
  }
  if (p.out_fp32) {                              // detection heads: cout = 3 (5 + C) need not be a multiple of 16
    for (int rep = 0; rep < nrep; ++rep) {
      float* o = static_cast<float*>(p.out) + (orow0 + (rep >> 1) * W2 + (rep & 1)) * p.out_ld + col0;
#pragma unroll
      for (int j = 0; j < 16; ++j)
        if (col0 + j < p.cout) o[j] = v[j];
    }
    return;
  }
  if constexpr (std::is_same<T, __nv_fp8_e4m3>::value) {
    // e4m3: residual codes times their buffer's scale, then value / s_out -> one 16-byte store of 16 codes per copy
    if (p.res != nullptr) {
      const uint4 u = __ldg(reinterpret_cast<const uint4*>(static_cast<const uint8_t*>(p.res) + orow0 * p.res_ld + col0));
      e4m3x16_unpack_fma(u, p.res_scale, v);
    }
    const uint4 pk = e4m3x16_pack(v, p.out_inv_scale);
    for (int rep = 0; rep < nrep; ++rep)
      *reinterpret_cast<uint4*>(static_cast<uint8_t*>(p.out) + (orow0 + (rep >> 1) * W2 + (rep & 1)) * p.out_ld + col0) = pk;
  } else {
    if (SRES || p.res != nullptr) {
      const uint4* rp = reinterpret_cast<const uint4*>(static_cast<const T*>(p.res) + orow0 * p.res_ld + col0);
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const uint4 u = SRES ? (j == 0 ? *sr0 : *sr1) : __ldg(rp + j);
        float2 f;
        f = Pack2<T>::unpack(u.x); v[8 * j + 0] += f.x; v[8 * j + 1] += f.y;
        f = Pack2<T>::unpack(u.y); v[8 * j + 2] += f.x; v[8 * j + 3] += f.y;
        f = Pack2<T>::unpack(u.z); v[8 * j + 4] += f.x; v[8 * j + 5] += f.y;
        f = Pack2<T>::unpack(u.w); v[8 * j + 6] += f.x; v[8 * j + 7] += f.y;
      }
    }
    uint4 pk[2];
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      pk[j].x = Pack2<T>::pack(v[8 * j + 0], v[8 * j + 1]);
      pk[j].y = Pack2<T>::pack(v[8 * j + 2], v[8 * j + 3]);
      pk[j].z = Pack2<T>::pack(v[8 * j + 4], v[8 * j + 5]);
      pk[j].w = Pack2<T>::pack(v[8 * j + 6], v[8 * j + 7]);
    }
    for (int rep = 0; rep < nrep; ++rep) {
      uint4* op = reinterpret_cast<uint4*>(static_cast<T*>(p.out) + (orow0 + (rep >> 1) * W2 + (rep & 1)) * p.out_ld + col0);
      op[0] = pk[0];
      op[1] = pk[1];
    }
  }
}

// Register epilogue (YB_CONV_EPI=reg): every thread stores its own accumulator fragments — two adjacent channels of
// rows r0 and r0 + 8 per 8-column block — straight to global memory, without the staging tile and its barriers.
template <typename T, int BN>
__device__ __forceinline__ void epilogue_reg(const ConvParams& p, const float (&acc)[BN / 2], const int row0, const int n0,
                                             const float* s_ss, const int t) {
  const int ncols = min(BN, p.cout - n0);
  const int rbase = row0 + 16 * (t >> 5) + ((t & 31) >> 2), cq = 2 * (t & 3);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = rbase + 8 * h;
    if (row >= p.M) continue;
    long orow[4] = {row, 0, 0, 0};
    int nrep = 1;
    if (p.upsample || p.scatter) {
      const int q = row % p.Q;
      const int pp = (row / p.Q) % p.P;
      const int img = row / (p.Q * p.P);
      const long W2 = 2L * p.Q;
      const long base = ((long)img * 2 * p.P + 2 * pp) * W2 + 2 * q;
      if (p.scatter) {
        orow[0] = base + ((p.scatter - 1) >> 1) * W2 + ((p.scatter - 1) & 1);
      } else {
        orow[0] = base; orow[1] = base + 1; orow[2] = base + W2; orow[3] = base + W2 + 1;
        nrep = 4;
      }
    }
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const int c = 8 * j + cq;                  // column inside the tile
      if (c >= ncols) continue;
      float v0 = fmaf(acc[4 * j + 2 * h], s_ss[c], s_ss[BN + c]);
      float v1 = fmaf(acc[4 * j + 2 * h + 1], s_ss[c + 1], s_ss[BN + c + 1]);
      if (p.leaky) { v0 = fmaxf(v0, 0.1f * v0); v1 = fmaxf(v1, 0.1f * v1); }
      const long col = n0 + c;
      if (p.out_fp32) {
        for (int rep = 0; rep < nrep; ++rep) {
          float* o = static_cast<float*>(p.out) + orow[rep] * p.out_ld + col;
          o[0] = v0;
          if (c + 1 < ncols) o[1] = v1;
        }
        continue;
      }
      if (p.res != nullptr) {
        const float2 r = Pack2<T>::unpack(*reinterpret_cast<const uint32_t*>(static_cast<const T*>(p.res) + orow[0] * p.res_ld + col));
        v0 += r.x; v1 += r.y;
      }
      const uint32_t pk = Pack2<T>::pack(v0, v1);
      for (int rep = 0; rep < nrep; ++rep)
        *reinterpret_cast<uint32_t*>(static_cast<T*>(p.out) + orow[rep] * p.out_ld + col) = pk;
    }
  }
}

// Detection-head epilogue with the decode fused in (yb_net_detect): instead of storing the fp32 feature map
// (model.py:55-58) for predict_kernel and nms_compact_kernel to re-read, every row — one grid cell, 3 anchors x
// E = 5 + C logits, all inside this n-tile — becomes 3 boxes (model.py:82-137, 182-188) and the (box, class) pairs with
// score = sigmoid(conf) * sigmoid(prob) >= thr (test_single_image.py:55, utils/nms_utils.py:30) are appended to the
// per-(image, class) candidate lists of the NMS (csrc/nms.cu).  Same arithmetic as predict_kernel (decode.cuh), so
// boxes and scores are bit-identical to the unfused path; the feature maps and the [n, B, C] score tensor never exist.
// The columns arrive chunk by chunk through the staging tile; threads 0..63 of the warpgroup (warps 0 and 1) own one
// row each and walk it anchor by anchor: the 5 box logits, then the C class logits, staging the next chunk when a column
// leaves the staged one.  A warp without a candidate for an anchor stages past its class logits without reading them.
// E = 5 + C is read at run time: one instantiation per tile width serves every class count whose 3 E columns fit it
// (conv_select).
template <int BN>
__device__ __forceinline__ void epilogue_detect(const ConvParams& p, const float (&acc)[BN / 2], const int row0, const int t,
                                                float* stg, const float* s_ss, const int bar_id) {
  const DetParams& d = p.det;
  const int E = d.E;
  const int lane = t & 31;
  const bool walker = t < WG_ROWS;                             // warp-uniform
  const int row = row0 + t;
  const bool row_ok = walker && row < p.M;
  const int cells = p.P * p.Q;
  const int img = row_ok ? row / cells : -1 - lane;            // rows past M: distinct dummies, never grouped, never stored
  const int cell = row_ok ? row - img * cells : 0;
  const unsigned same = __match_any_sync(0xffffffffu, img);   // lanes of my image (candidate slots are reserved per image)
  const unsigned lt = (1u << lane) - 1u;
  const float offx = (float)(cell % p.Q), offy = (float)(cell / p.Q);
  const int box0 = d.box_off + cell * 3;
  const int NCH = (3 * E + 31) / 32;
  // chunk ch of the accumulator block -> the staging tile (every thread of the warpgroup, chunks in increasing order)
  auto stage = [&](int ch) {
    warpgroup_bar(bar_id);                                     // the previous chunk's readers are done with the tile
    wgmma_stage_chunk<BN>(acc, ch, stg, EPI_LD, t);
    warpgroup_bar(bar_id);
  };
  if (!walker) {                                               // warps 2 and 3 only help stage
#pragma unroll 1
    for (int ch = 0; ch < NCH; ++ch) stage(ch);
    return;
  }
  const float* myrow = stg + t * EPI_LD;
  int staged = -1;                                             // the chunk in the staging tile
  // logit of tile column col (col <= 32 (staged + 1)): its chunk is staged first if it is not there yet
  auto logit = [&](int col) -> float {
    if ((col >> 5) != staged) stage(++staged);
    return fmaf(myrow[col & 31], s_ss[col], s_ss[BN + col]);   // scale 1, shift = bias
  };
#pragma unroll 1
  for (int a = 0; a < 3; ++a) {
    const int c0 = a * E;                                      // x, y, w, h, conf, then the C class logits
    const float h0 = logit(c0), h1 = logit(c0 + 1), h2 = logit(c0 + 2), h3 = logit(c0 + 3);
    const float cconf = sigmoid_ref(logit(c0 + 4));            // model.py:167
    const bool cok = row_ok && cconf >= d.thr;                 // score = conf * prob <= conf: nothing below thr can pass
    if (row_ok) {
      float4 b;
      decode_axis(h0, h2, offx, d.ratio_w, d.anchor_w[a], b.x, b.z);
      decode_axis(h1, h3, offy, d.ratio_h, d.anchor_h[a], b.y, b.w);
      reinterpret_cast<float4*>(d.boxes)[(long)img * d.B + box0 + a] = b;
    }
    if (!__any_sync(0xffffffffu, cok)) {                       // no candidate in this warp: stage past the class logits
      while (staged < (c0 + E - 1) >> 5) stage(++staged);
      continue;
    }
#pragma unroll 1
    for (int c = 0; c < d.C; ++c) {
      const float v = logit(c0 + 5 + c);
      bool pass = false;
      float sc = 0.f;
      if (cok && v >= d.logit_lo) {
        sc = __fmul_rn(cconf, sigmoid_ref(v));                 // model.py:168, test_single_image.py:55
        pass = sc >= d.thr;                                    // utils/nms_utils.py:30
      }
      const unsigned m = __ballot_sync(0xffffffffu, pass);
      if (m != 0u) {                                           // warp-uniform
        const unsigned mine = m & same;
        const int leader = pass ? __ffs(mine) - 1 : lane;
        int base = 0;
        if (pass && lane == leader) base = atomicAdd(d.cand_count + img * d.C + c, __popc(mine));
        base = __shfl_sync(0xffffffffu, base, leader);
        if (pass) {
          const long seg = ((long)img * d.C + c) * d.B;
          const int slot = base + __popc(mine & lt);
          d.cand_score[seg + slot] = sc;
          d.cand_idx[seg + slot] = box0 + a;
        }
      }
    }
  }
}

// TMA-store epilogue (TMA, 16-bit plain outputs; conv_select): the values never leave the accumulator layout.  Each
// warp owns 16 rows of a 64-row accumulator block, so it works alone, without a warpgroup barrier: per 64-column box it
// applies scale / shift (+leaky) (+residual) to its fragments in registers — the operations of epi_store16 in the
// same order, so the outputs are the same bit for bit — packs them to 16 bits, writes them with four stmatrix.x4 into
// a 16-row x 64-column slab of 128-byte rows in the TMA's 128B swizzle (conflict-free; epi_box_to_slab, wgmma.cuh),
// and lane 0 stores the slab through p.tmO, which clips rows >= M and columns >= cout.
//   ss4[4 j + q]: (scale, scale, shift, shift) of columns 8 j + 2 q and + 1 of the tile.
//   Without RES the warp has one slab (slab_h = slab_b = 0) and waits until the previous store has read it; such a
//   launch has no residual (conv_select: a residual that is not prefetched keeps the staged epilogue).
//   RES: the slab of block h, box b is the warp's 16 rows of the shortcut tile itself (slab + h slab_h + b slab_b),
//   already in that layout: ldmatrix.x4 reads the residual as fragments and the result goes back over it.
// acc: [NH][BN / 2]; row0: the first of the warp's 16 rows in block 0 (block h: + 64 h).
template <typename T, int BN, int NH, bool RES>
__device__ __forceinline__ void epilogue_tma(const ConvParams& p, const float (&acc)[NH][BN / 2], const int row0,
                                             const int n0, const float4* ss4, uint8_t* slab, const uint32_t slab_h,
                                             const uint32_t slab_b, const int lane) {
  const float slope = p.leaky ? 0.1f : 1.f;                    // fmaxf(v, 1 v) == v
#pragma unroll
  for (int h = 0; h < NH; ++h) {
#pragma unroll
    for (int b = 0; b < BN / 64; ++b) {
      uint8_t* s = slab + h * slab_h + b * slab_b;
      epi_box_to_slab<T, BN, RES>(acc[h], b, ss4, s, slope, lane);
      if (lane == 0 && row0 + h * WG_ROWS < p.M && n0 + b * 64 < p.cout) {
        tma_store_2d(&p.tmO, s, n0 + b * 64, row0 + h * WG_ROWS);
        bulk_commit_group();
      }
    }
  }
}

// named barriers (0 = __syncthreads; 1, 2 = the consumer warpgroups' own barriers): MMA_TURN + w = "warpgroup w may
// start its next main loop" (ping-pong)
static constexpr int MMA_TURN_BAR = 3;

// DET: detection head with the decode fused in (epilogue_detect), all 3 (5 + C) columns in the one n-tile.  PP:
// ping-pong schedule (NC = 2, staged epilogue, no fused decode; see the top of the file).  BKB: bytes per k-block row (Cfg).
// CM x CN: a cluster of CM m-tiles x CN n-tiles, both schedules.  Each CTA loads 1/CN of its A tile, multicast to the
// CN CTAs of its m-tile, and 1/CM of its B tile, multicast to the CM CTAs of its n-tile: every CTA still receives the
// full STAGE_BYTES per k-block but reads only A_BYTES / CN + B_BYTES / CM of them from L2.  Each warpgroup computes
// the same tiles with the same wgmma sequence as without the cluster, so the outputs are the same bit for bit.
// CM = 0 (the cooperative launches): a p.cluster x 1 cluster, the shape read at run time, so that one instantiation
// serves the YB_CONV_MODE clusters.  The ping-pong launches, which the inference plans cluster, keep the shape in the
// template: as a run-time shape it cost their 3x3 layers 2-3 % (DESIGN.md §5).
// RES (ping-pong, 16-bit, p.res != nullptr, YB_CONV_RES): the shortcut tile of every work unit is prefetched by TMA
// (p.tmR) into its warpgroup's shared-memory tile while the unit's main loop runs, and the epilogue adds it from there
// instead of waiting on a global load per 32-column chunk.  Each CTA loads its own tile (never multicast).
// TMA (16-bit, NC = 2, no fused decode; p.epi_tma): the TMA-store epilogue (epilogue_tma) in place of the staged one.
// The warps' output slabs lie where the staging tiles would; with RES they are the shortcut tile itself.
template <typename T, int BN, int BKB, int NC, bool DET = false, bool PP = false, int CM = 0, int CN = 1, bool RES = false,
          bool TMA = false>
__global__ void __launch_bounds__(128 * (NC + 1), 1)
conv_igemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                  const __grid_constant__ ConvParams p) {
  static_assert(!PP || (NC == 2 && !DET), "ping-pong: two consumer warpgroups, no fused decode");
  static_assert(!RES || (PP && sizeof(T) == 2), "the shared-memory shortcut tile is a 16-bit ping-pong variant");
  static_assert(CM != 0 || CN == 1, "a run-time cluster shape is p.cluster x 1");
  static_assert(!TMA || (sizeof(T) == 2 && NC == 2 && !DET), "the TMA-store epilogue: 16-bit, 128-row tiles, no fused decode");
  constexpr int NH = PP ? 2 : 1;                         // 64-row accumulator blocks per consumer warpgroup
  using C = Cfg<BN, BKB, NC, RES>;
  constexpr int BK = BKB / (int)sizeof(T);               // channels per k-block
  extern __shared__ uint8_t smem_raw[];
  // 1024-byte alignment by POINTER ARITHMETIC on the __shared__ array: an integer round trip makes the pointer generic,
  // and every staging-tile access then compiles to generic loads / stores instead of LDS / STS
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* sA = smem;
  uint8_t* sB = smem + C::STAGES * C::A_BYTES;
  uint8_t* sR = smem + C::STAGES * C::STAGE_BYTES;       // RES: [NC] shortcut tiles, 1024-byte aligned
  float* s_epi = reinterpret_cast<float*>(sR + C::RES_BYTES);   // [NC][64][EPI_LD] staging tiles
  float* s_stat = s_epi + NC * EPI_FLOATS;               // [NC][2][BN] per-CTA column sums / sums of squares
  float* s_ss = s_stat + NC * 2 * BN;                    // [NC][2][BN] scale / shift of each warpgroup's current n-tile
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(s_ss + NC * 2 * BN);   // [STAGES] TMA -> MMA
  uint64_t* empty_bar = full_bar + 8;                    // [STAGES] MMA -> TMA: one arrive per consumer warp of the cluster
                                                         // (ping-pong: of the one warpgroup that read the stage)
  uint64_t* res_full = empty_bar + 8;                    // RES: [NC] shortcut tile landed
  uint64_t* res_empty = res_full + NC;                   // RES: [NC] the warpgroup's epilogue has read it (4 warps)

  // warp-uniform by construction: ptxas then keeps the ping-pong consumer's 128 accumulators out of local memory
  const int wg = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 7), 0);
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int i = 0; i < C::STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      // every consumer warp that reads a stage arrives on that stage's empty barrier in every CTA of the cluster (any of
      // them may multicast into it next): ping-pong, the 4 warps of the one warpgroup that read it
      mbar_init(&empty_bar[i], 4 * (PP ? 1 : NC) * (CM ? CM * CN : p.cluster));
    }
    if constexpr (TMA) tma_prefetch_desc(&p.tmO);
    if constexpr (RES) {
      tma_prefetch_desc(&p.tmR);
      for (int i = 0; i < NC; ++i) {
        mbar_init(&res_full[i], 1);
        mbar_init(&res_empty[i], 4);
      }
    }
    fence_barrier_init();
  }
  __syncthreads();
  if (p.cluster > 1) cluster_sync_all();                 // every peer's barriers exist before the first multicast

  const int cm = CM ? CM : p.cluster;                    // cluster shape cm x CN
  const int cs = cm * CN;                                // CTAs per cluster (1: no cluster, no multicast)
  const uint32_t rank = cs > 1 ? cluster_ctarank() : 0u;
  const int cluster_id = blockIdx.x / cs, num_clusters = gridDim.x / cs;
  const int nunits = num_units<CM, CN>(p);
  const int kb_per_tap = p.cin / BK;
  const int num_kb = p.kh * p.kw * kb_per_tap;

  if (wg == 0) {
    // ===================== TMA producer =====================
    // One thread runs the whole loop: a k-block costs one barrier wait, one expect_tx and two TMA issues.  The filter
    // tap / channel-chunk coordinates are carried as counters instead of being divided out of the k-block index.
    // CTA (rm, rn) of a cm x CN cluster loads A rows [rn BLOCK_M / CN, +BLOCK_M / CN) — for a 3x3 conv an im2col box of
    // BLOCK_M / CN pixels from output pixel m0 + rn BLOCK_M / CN — multicast to the CTAs (rm, *), and B rows
    // [rm BN / cm, +BN / cm), multicast to the CTAs (*, rn); a load with one destination is a plain TMA load.  The
    // slices start on whole 8-row swizzle groups, so they land exactly where the whole-tile loads put them.
    if (threadIdx.x == 0) {
      const int a_rows = C::BLOCK_M / CN, b_rows = BN / cm;
      const int rm = (int)rank / CN, rn = (int)rank % CN;
      const uint16_t a_mask = (uint16_t)(((1u << CN) - 1u) << (rm * CN));
      uint16_t b_mask = 0;
      for (int i = 0; i < cm; ++i) b_mask |= (uint16_t)(1u << (i * CN + rn));
      int stage = 0;
      uint32_t phase = 0;
      for (int unit = cluster_id; unit < nunits; unit += num_clusters) {
        int m_idx, n_idx;
        unit_coords<CM, CN>(p, unit, rank, m_idx, n_idx);
        const int ma = m_idx * C::BLOCK_M + rn * a_rows;       // first row of this CTA's A slice
        const int nb = n_idx * BN + rm * b_rows;               // first row of this CTA's B slice
        // first output pixel of the slice -> (image, row, col); base input pixel of the filter window
        const int q = ma % p.Q;
        const int pp = (ma / p.Q) % p.P;
        const int img = ma / (p.Q * p.P);
        const int w_base = q * p.stride - p.pad;
        const int h_base = pp * p.stride - p.pad;
        int c0 = 0, tw = 0, th = 0, kcol = 0;                  // channel chunk, tap (tw, th), column in the packed weights
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          mbar_arrive_expect_tx(&full_bar[stage], C::STAGE_BYTES);
          uint8_t* a_dst = sA + stage * C::A_BYTES + rn * a_rows * BKB;
          uint8_t* b_dst = sB + stage * C::B_BYTES + rm * b_rows * BKB;
          if constexpr (CN > 1) {
            if (p.im2col)
              tma_load_im2col_4d_multicast(a_dst, &tmA, &full_bar[stage], c0, w_base, h_base, img, (uint16_t)tw,
                                           (uint16_t)th, a_mask);
            else
              tma_load_2d_multicast(a_dst, &tmA, &full_bar[stage], c0, ma, a_mask);
          } else {
            if (p.im2col)
              tma_load_im2col_4d(a_dst, &tmA, &full_bar[stage], c0, w_base, h_base, img, (uint16_t)tw, (uint16_t)th);
            else
              tma_load_2d(a_dst, &tmA, &full_bar[stage], c0, ma);
          }
          if (cm > 1) tma_load_2d_multicast(b_dst, &tmB, &full_bar[stage], kcol, nb, b_mask);
          else tma_load_2d(b_dst, &tmB, &full_bar[stage], kcol, nb);
          c0 += BK; kcol += BK;
          if (c0 == p.cin) { c0 = 0; if (++tw == p.kw) { tw = 0; ++th; } }
          if (++stage == C::STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
    if constexpr (RES) {
      // Shortcut tiles: one thread of warp 1 walks the CTA's units in the same order and loads unit j's tile into
      // warpgroup (j & 1)'s buffer as soon as that warpgroup's epilogue has released the tile of its previous unit, so
      // the load has the whole main loop of unit j to land.  Independent of the operand ring: the ring never waits on
      // an epilogue.  Units wholly past M (cluster ranks past the last m-tile) have nothing to add and are skipped on
      // both sides.
      if (threadIdx.x == 32) {
        uint32_t rphase[NC] = {};
        int j = 0;
        for (int unit = cluster_id; unit < nunits; unit += num_clusters, ++j) {
          int m_idx, n_idx;
          unit_coords<CM, CN>(p, unit, rank, m_idx, n_idx);
          const int m0 = m_idx * C::BLOCK_M, n0 = n_idx * BN;
          if (m0 >= p.M) continue;
          const int w = j & 1;
          mbar_wait(&res_empty[w], rphase[w] ^ 1);
          mbar_arrive_expect_tx(&res_full[w], C::RES_TILE_BYTES);
#pragma unroll
          for (int b = 0; b < BN / C::RES_BOX_COLS; ++b)
            tma_load_2d(sR + w * C::RES_TILE_BYTES + b * C::RES_BOX_BYTES, &p.tmR, &res_full[w], n0 + b * C::RES_BOX_COLS, m0);
          rphase[w] ^= 1;
        }
      }
    }
  } else {
    // ===================== MMA + epilogue =====================
    // cooperative: warpgroup cw computes rows [64 cw, 64 cw + 64) of every tile of the CTA;
    // ping-pong: warpgroup cw computes all 128 rows of every other tile of the CTA (its j-th unit is the CTA's 2j + cw-th)
    using Mma = typename ConvMma<T, BN>::type;
    constexpr bool kRegEpi = !PP && !TMA && !std::is_same<T, __nv_fp8_e4m3>::value;   // YB_CONV_EPI=reg: 16-bit only
    const int cw = wg - 1;
    const int t = threadIdx.x & 127;
    const int lane = t & 31;
    const int bar_id = 1 + cw;
    float* stg = s_epi + cw * EPI_FLOATS;
    float* sst = s_stat + cw * 2 * BN;
    float* sss = s_ss + cw * 2 * BN;
    if (p.stat_sum != nullptr)
      for (int c = t; c < 2 * BN; c += 128) sst[c] = 0.f;   // (first read after the scale / shift barriers below)
    // a stage is released on the empty barrier of every CTA of the cluster: any of them may multicast into it next
    // (unrolled over the largest cluster: no loop in the k-loop when the shape is a run-time one)
    auto release = [&](int st) {
      __syncwarp();
      if (lane == 0) {
        if (cs == 1) {
          mbar_arrive(&empty_bar[st]);
        } else {
#pragma unroll
          for (int r = 0; r < 4; ++r)
            if (r < cs) mbar_arrive_remote(&empty_bar[st], (uint32_t)r);
        }
      }
    };
    float acc[NH][BN / 2];
    int stage = 0, prev = 0;
    uint32_t phase = 0;
    // ping-pong: step the ring position over the other warpgroup's unit (the producer fills the ring in unit order)
    auto skip_unit = [&]() {
      const int s = stage + num_kb;
      phase ^= (uint32_t)((s / C::STAGES) & 1);
      stage = s % C::STAGES;
    };
    if (PP && cw == 1) skip_unit();
    int cur_n0 = -1, ss_n0 = -1;
    const uint32_t a_off = PP ? 0u : cw * WG_ROWS * BKB;
    const int unit_step = PP ? 2 * num_clusters : num_clusters;
    uint32_t res_phase = 0;
    const uint8_t* sres = sR + cw * C::RES_TILE_BYTES;   // RES: this warpgroup's shortcut tile
    for (int unit = cluster_id + (PP ? cw * num_clusters : 0); unit < nunits; unit += unit_step) {
      int m_idx, n_idx;
      unit_coords<CM, CN>(p, unit, rank, m_idx, n_idx);
      const int m0 = m_idx * C::BLOCK_M;
      const int n0 = n_idx * BN;
      // Ping-pong: wait until the other warpgroup has issued the previous unit's main loop.  Besides keeping the two
      // main loops from interleaving on the tensor cores, this makes every fill of the ring before this unit's
      // complete, so a parity wait below cannot match a fill two phases old.
      if (PP && unit != cluster_id) named_bar_sync(MMA_TURN_BAR + cw, 256);
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t a_addr = smem_u32(sA + stage * C::A_BYTES) + a_off;
        const uint32_t b_addr = smem_u32(sB + stage * C::B_BYTES);
#pragma unroll
        for (int h = 0; h < NH; ++h) wgmma_fence_operand(acc[h]);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BKB / 32; ++k)
#pragma unroll
          for (int h = 0; h < NH; ++h)
            Mma::mma(acc[h], make_kmajor_desc(a_addr + h * WG_ROWS * BKB + k * 32, C::SBO, C::SWIZZLE),
                     make_kmajor_desc(b_addr + k * 32, C::SBO, C::SWIZZLE), (kb | k) != 0);
        wgmma_commit();
#pragma unroll
        for (int h = 0; h < NH; ++h) wgmma_fence_operand(acc[h]);
        wgmma_wait<1>();                         // the previous k-block's MMAs have retired: its stage is free
        if (kb > 0) release(prev);
        prev = stage;
        if (++stage == C::STAGES) { stage = 0; phase ^= 1; }
      }
      if (PP && unit + num_clusters < nunits) named_bar_arrive(MMA_TURN_BAR + (cw ^ 1), 256);   // the other's turn
      wgmma_wait<0>();
#pragma unroll
      for (int h = 0; h < NH; ++h) wgmma_fence_operand(acc[h]);
      release(prev);
      if (PP) skip_unit();

      if (p.stat_sum != nullptr && n0 != cur_n0) {
        if (cur_n0 >= 0) stat_flush<BN>(p, sst, cur_n0, t, bar_id);
        cur_n0 = n0;
      }
      if (n0 != ss_n0) {
        warpgroup_bar(bar_id);                   // nobody still reads the previous n-tile's values
        for (int c = t; c < BN; c += 128) {
          // scale = shift = NULL: identity (dgrad convs).  A fused-decode head's tile may be wider than its cout_pad
          // parameters (C 38-59: 192 on a 256-column tile); it reads only its first cout = 3 E columns.
          const bool in = !DET || c < p.cout;
          const float sc = p.scale && in ? __ldg(p.scale + n0 + c) : 1.f;
          const float sh = p.shift && in ? __ldg(p.shift + n0 + c) : 0.f;
          if constexpr (TMA) {                   // (scale, scale, shift, shift) per column pair: one load per fragment
            sss[(c >> 1) * 4 + (c & 1)] = sc;
            sss[(c >> 1) * 4 + 2 + (c & 1)] = sh;
          } else {
            sss[c] = sc;
            sss[BN + c] = sh;
          }
        }
        warpgroup_bar(bar_id);
        ss_n0 = n0;
      }
      if constexpr (DET) {
        epilogue_detect<BN>(p, acc[0], m0 + cw * WG_ROWS, t, stg, sss, bar_id);
      } else if constexpr (TMA) {
        if (m0 < p.M) {                          // units wholly past M store nothing
          const int wrow = 16 * (t >> 5);        // this warp's rows of each 64-row block
          const int row0 = m0 + (PP ? 0 : cw * WG_ROWS) + wrow;
          if constexpr (RES) {
            mbar_wait(&res_full[cw], res_phase);
            epilogue_tma<T, BN, NH, true>(p, acc, row0, n0, reinterpret_cast<const float4*>(sss),
                                          sR + cw * C::RES_TILE_BYTES + wrow * 128, WG_ROWS * 128, C::RES_BOX_BYTES, lane);
            // the stores have read the warp's rows of the tile: the producer may refill it
            if (lane == 0) {
              bulk_wait_group_read<0>();
              mbar_arrive(&res_empty[cw]);
            }
            res_phase ^= 1;
          } else {
            epilogue_tma<T, BN, NH, false>(p, acc, row0, n0, reinterpret_cast<const float4*>(sss),
                                           reinterpret_cast<uint8_t*>(s_epi) + (cw * 4 + (t >> 5)) * 2048, 0, 0, lane);
          }
        }
      } else if (kRegEpi && p.epi_reg) {
        if constexpr (kRegEpi) epilogue_reg<T, BN>(p, acc[0], m0 + cw * WG_ROWS, n0, sss, t);
      } else {
        // the accumulator blocks as one row of NH * BN / 32 chunks: one copy of the epilogue serves both halves
        const float(&acc_all)[NH * BN / 2] = reinterpret_cast<const float(&)[NH * BN / 2]>(acc);
        const int nvalid = min(BN / 32, (p.cout - n0 + 31) >> 5);   // zero-padded weight rows (cout_pad > cout): not stored
        const int er = t >> 1, eh = t & 1;       // this thread's row of the chunk and its 16-column half
        if constexpr (RES) {
          if (m0 < p.M) mbar_wait(&res_full[cw], res_phase);
        }
#pragma unroll 1
        for (int h = 0; h < NH; ++h) {
          const int row0 = m0 + (PP ? h : cw) * WG_ROWS;
#pragma unroll 1
          for (int ch = 0; ch < nvalid; ++ch) {
            warpgroup_bar(bar_id);               // the previous chunk's readers are done with the staging tile
            wgmma_stage_chunk<NH * BN>(acc_all, h * (BN / 32) + ch, stg, EPI_LD, t);
            warpgroup_bar(bar_id);
            if (p.stat_sum != nullptr) {         // BN batch statistics of the raw conv output: lane = column
              const int col = t & 31, rg = (t >> 5) * 16;
              float cs_ = 0.f, cs2 = 0.f;
#pragma unroll 4
              for (int rr = 0; rr < 16; ++rr) {
                if (row0 + rg + rr < p.M) {
                  const float v = stg[(rg + rr) * EPI_LD + col];
                  cs_ += v;
                  cs2 = fmaf(v, v, cs2);
                }
              }
              atomicAdd(&sst[ch * 32 + col], cs_);
              atomicAdd(&sst[BN + ch * 32 + col], cs2);
            }
            if (row0 + er < p.M) {
              const int cl = ch * 32 + eh * 16;
              if constexpr (RES) {
                // row rl of the tile, columns cl..cl+15 = 16-byte chunks c, c+1 of a 128-byte row of box cl / 64,
                // stored at chunk ^ (rl & 7) (TMA 128B swizzle)
                const int rl = h * WG_ROWS + er, c = (cl % C::RES_BOX_COLS) >> 3;
                const uint8_t* rrow = sres + (cl / C::RES_BOX_COLS) * C::RES_BOX_BYTES + rl * 128;
                epi_store16<T, true>(p, stg + er * EPI_LD + eh * 16, row0 + er, n0 + cl, sss + cl, sss + BN + cl,
                                     reinterpret_cast<const uint4*>(rrow + ((c ^ (rl & 7)) << 4)),
                                     reinterpret_cast<const uint4*>(rrow + (((c + 1) ^ (rl & 7)) << 4)));
              } else {
                epi_store16<T>(p, stg + er * EPI_LD + eh * 16, row0 + er, n0 + cl, sss + cl, sss + BN + cl);
              }
            }
          }
        }
        if constexpr (RES) {
          if (m0 < p.M) {                        // this warp's last read of the tile is done: the producer may refill it
            __syncwarp();
            if (lane == 0) mbar_arrive(&res_empty[cw]);
            res_phase ^= 1;
          }
        }
      }
    }
    if (p.stat_sum != nullptr && cur_n0 >= 0) stat_flush<BN>(p, sst, cur_n0, t, bar_id);
    if constexpr (TMA) {
      if (lane == 0) bulk_wait_group<0>();       // this warp's output stores are complete before the CTA may exit
    }
  }
  if (cs > 1) cluster_sync_all();                        // no CTA exits while a peer may still multicast into it or arrive on it
}

// ----------------------------------------------------------------------------------
// host: tensor maps (driver entry points fetched at run time: no link-time libcuda)
// ----------------------------------------------------------------------------------
static PFN_cuTensorMapEncodeTiled_v12000 g_encode_tiled = nullptr;
static PFN_cuTensorMapEncodeIm2col_v12000 g_encode_im2col = nullptr;

static int load_driver_entry_points() {
  if (g_encode_tiled && g_encode_im2col) return YB_OK;
  cudaDriverEntryPointQueryResult qr;
  void* fn = nullptr;
  YB_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qr));
  if (qr != cudaDriverEntryPointSuccess || !fn) { set_error("cuTensorMapEncodeTiled not available"); return YB_ERR_CUDA; }
  g_encode_tiled = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(fn);
  YB_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &fn, cudaEnableDefault, &qr));
  if (qr != cudaDriverEntryPointSuccess || !fn) { set_error("cuTensorMapEncodeIm2col not available"); return YB_ERR_CUDA; }
  g_encode_im2col = reinterpret_cast<PFN_cuTensorMapEncodeIm2col_v12000>(fn);
  return YB_OK;
}

static CUtensorMapDataType tm_dtype(int dtype) {
  if (dtype == YB_E4M3) return CU_TENSOR_MAP_DATA_TYPE_UINT8;
  return dtype == YB_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
}
static int tm_esize(int dtype) { return dtype == YB_E4M3 ? 1 : 2; }

// 2D row-major [rows, cols] 16-bit / e4m3 matrix, row pitch `ld` elements; box = [box_rows, box_cols]
int make_tmap_2d(CUtensorMap* tm, const void* base, int dtype, long rows, long cols, long ld, int box_rows,
                 int box_cols, int weights) {
  int rc = load_driver_entry_points();
  if (rc) return rc;
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  const int es = tm_esize(dtype);
  cuuint64_t strides[1] = {(cuuint64_t)ld * es};
  cuuint32_t box[2] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUtensorMapSwizzle sw = box_cols * es == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B;
  CUresult r = g_encode_tiled(tm, tm_dtype(dtype), 2, const_cast<void*>(base), dims, strides, box, estr,
                              CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                              weights ? CU_TENSOR_MAP_L2_PROMOTION_L2_256B : CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (%d): rows=%ld cols=%ld ld=%ld box=%dx%d", (int)r, rows, cols, ld,
              box_rows, box_cols);
    return YB_ERR_CUDA;
  }
  return YB_OK;
}

// float32 image [n, h, w, 3] seen as {W*3, H, N}: box = box_f floats x box_h rows of one image, no swizzle, zero fill
// outside (the fused stem's input halo, csrc/conv_halo.cu).  w*3*4 bytes must be a multiple of 16 (w % 4 == 0).
int make_tmap_image3d(CUtensorMap* tm, const float* base, int n, int h, int w, int box_f, int box_h) {
  int rc = load_driver_entry_points();
  if (rc) return rc;
  cuuint64_t dims[3] = {(cuuint64_t)w * 3, (cuuint64_t)h, (cuuint64_t)n};
  cuuint64_t strides[2] = {(cuuint64_t)w * 3 * 4, (cuuint64_t)h * w * 3 * 4};
  cuuint32_t box[3] = {(cuuint32_t)box_f, (cuuint32_t)box_h, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = g_encode_tiled(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(base), dims, strides, box, estr,
                              CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled(image) failed (%d): n=%d h=%d w=%d box=%dx%d", (int)r, n, h, w, box_f, box_h);
    return YB_ERR_CUDA;
  }
  return YB_OK;
}

// NHWC activation seen as {C, W, H, N}, TILED mode: box = box_c channels x box_w x box_h pixels of one image, traversal
// stride `estride` along W and H (a box spanning 2 * count - 1 pixels at stride 2 loads `count` of them); pixels outside
// the image come back zero-filled.  Used by the halo-tile conv (csrc/conv_halo.cu).
int make_tmap_tiled4d(CUtensorMap* tm, const void* base, int dtype, int n, int h, int w, int c, long ld, int box_c,
                      int box_w, int box_h, int estride) {
  int rc = load_driver_entry_points();
  if (rc) return rc;
  cuuint64_t dims[4] = {(cuuint64_t)c, (cuuint64_t)w, (cuuint64_t)h, (cuuint64_t)n};
  cuuint64_t strides[3] = {(cuuint64_t)ld * 2, (cuuint64_t)w * ld * 2, (cuuint64_t)h * w * ld * 2};
  cuuint32_t box[4] = {(cuuint32_t)box_c, (cuuint32_t)box_w, (cuuint32_t)box_h, 1};
  cuuint32_t estr[4] = {1, (cuuint32_t)estride, (cuuint32_t)estride, 1};
  CUtensorMapSwizzle sw = box_c * 2 == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B;
  CUresult r = g_encode_tiled(tm, tm_dtype(dtype), 4, const_cast<void*>(base), dims, strides, box, estr,
                              CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled(4d) failed (%d): n=%d h=%d w=%d c=%d ld=%ld box=%dx%dx%d stride %d", (int)r, n, h, w, c,
              ld, box_c, box_w, box_h, estride);
    return YB_ERR_CUDA;
  }
  return YB_OK;
}

// NHWC activation seen as {C, W, H, N}; im2col traversal for a ksize x ksize window with
// symmetric padding `pad` and traversal stride `stride`; one request = 128 pixels x bk channels.
int make_tmap_im2col_px(CUtensorMap* tm, const void* base, int dtype, int n, int h, int w, int c, long ld, int ksize,
                        int stride, int pad, int bk, int pixels);
int make_tmap_im2col(CUtensorMap* tm, const void* base, int dtype, int n, int h, int w, int c, long ld, int ksize,
                     int stride, int pad, int bk) {
  return make_tmap_im2col_px(tm, base, dtype, n, h, w, c, ld, ksize, stride, pad, bk, 128);
}
// `pixels` = output pixels gathered per request (rows of the shared-memory box)
int make_tmap_im2col_px(CUtensorMap* tm, const void* base, int dtype, int n, int h, int w, int c, long ld, int ksize,
                        int stride, int pad, int bk, int pixels) {
  int rc = load_driver_entry_points();
  if (rc) return rc;
  cuuint64_t dims[4] = {(cuuint64_t)c, (cuuint64_t)w, (cuuint64_t)h, (cuuint64_t)n};
  const int es = tm_esize(dtype);
  cuuint64_t strides[3] = {(cuuint64_t)ld * es, (cuuint64_t)w * ld * es, (cuuint64_t)h * w * ld * es};
  // base-pixel bounding box: [-pad, dim-1 + pad-(k-1)]  (cutlass conv/collective/detail.hpp fprop rule)
  int lower[2] = {-pad, -pad};
  int upper[2] = {pad - (ksize - 1), pad - (ksize - 1)};
  cuuint32_t estr[4] = {1, (cuuint32_t)stride, (cuuint32_t)stride, 1};
  CUtensorMapSwizzle sw = bk * es == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B;
  CUresult r = g_encode_im2col(tm, tm_dtype(dtype), 4, const_cast<void*>(base), dims, strides, lower, upper,
                               (cuuint32_t)bk, (cuuint32_t)pixels, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                               CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeIm2col failed (%d): n=%d h=%d w=%d c=%d ld=%ld k=%d s=%d", (int)r, n, h, w, c, ld,
              ksize, stride);
    return YB_ERR_CUDA;
  }
  // Driver workaround used by CUTLASS (copy_traits_sm90_im2col.hpp): for tensors < 128 KiB
  // drivers <= 13.1 set a descriptor bit that makes the im2col traversal fault.
  int drv = 0;
  cudaDriverGetVersion(&drv);
  if (drv <= 13010 && (size_t)n * h * w * ld * es < 131072) {
    reinterpret_cast<uint64_t*>(tm)[1] &= ~(1ull << 21);
  }
  return YB_OK;
}

// the host's count of num_units
int conv_units(const ConvParams& p) {
  return ceil_div(p.num_m_tiles, p.cluster / p.cluster_n) * (p.num_n_tiles / p.cluster_n);
}

// Persistent grid in CTAs: one cluster per work unit, at most one CTA per SM and at most max_clusters resident clusters
// (cudaOccupancyMaxActiveClusters: an H100's GPCs hold 30, not 33, clusters of 4 of these CTAs), and at most p.ctas
// CTAs (rounded down to whole clusters, at least one cluster) when YB_CONV_CTAS caps it.
int conv_grid(const ConvParams& p, int sms, int max_active) {
  const int cs = p.cluster;
  const int units = conv_units(p);
  int max_clusters = sms / cs;
  if (max_active > 0 && max_active < max_clusters) max_clusters = max_active;
  if (p.ctas > 0) {
    const int cap = p.ctas / cs > 1 ? p.ctas / cs : 1;
    if (cap < max_clusters) max_clusters = cap;
  }
  const int clusters = units < max_clusters ? units : max_clusters;
  return clusters * cs;
}

// Most clusters of cs CTAs of `kern` resident at once on the current device, queried once per device and cluster size.
struct ClusterCapacity { int v[64][5] = {}; };
static int cluster_capacity(ClusterCapacity& cap, const void* kern, int threads, int smem, int cs, int* out) {
  int dev = 0;
  YB_CUDA(cudaGetDevice(&dev));
  int& v = cap.v[dev & 63][cs];
  if (v == 0) {
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3(cs);
    cfg.blockDim = dim3(threads);
    cfg.dynamicSmemBytes = smem;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = cs; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    int n = 0;
    YB_CUDA(cudaOccupancyMaxActiveClusters(&n, kern, &cfg));
    if (n <= 0) { set_error("conv: no cluster of %d CTAs (%d bytes of shared memory each) fits the device", cs, smem); return YB_ERR_CUDA; }
    v = n;
  }
  *out = v;
  return YB_OK;
}

// One conv_igemm_kernel instantiation: the type conv_kernel_for passes to its functor
template <typename T, int BN, int BKB, int NC, bool DET = false, bool PP = false, int CM = 0, int CN = 1, bool RES = false,
          bool TMA = false>
struct ConvKernel {
  using C = Cfg<BN, BKB, NC, RES>;
  static constexpr auto kernel = conv_igemm_kernel<T, BN, BKB, NC, DET, PP, CM, CN, RES, TMA>;
};

static int no_conv_kernel(const ConvParams& p) {
  set_error("conv: no kernel for dtype %d, %d-column tiles, %d-byte k-blocks, %d consumer warpgroups, ping-pong %d, "
            "%d x %d cluster, shortcut tile %d, TMA-store epilogue %d, fused decode of %d columns", p.dtype, p.block_n,
            p.block_kb, p.consumers, p.pingpong, p.cluster / p.cluster_n, p.cluster_n, p.res_smem, p.epi_tma, p.det_e);
  return YB_ERR_UNSUPPORTED;
}

// ping-pong: the cluster shape (cluster / cluster_n) x cluster_n is a template parameter; e4m3 runs unclustered
template <typename T, int BN, int BKB, bool RES, bool TMA, typename F>
static int conv_kernel_pp_shape(const ConvParams& p, F& f) {
  const int cn = p.cluster_n, cm = p.cluster / p.cluster_n;
  if (cm == 1 && cn == 1) return f(ConvKernel<T, BN, BKB, 2, false, true, 1, 1, RES, TMA>());
  if constexpr (sizeof(T) == 2) {
    if (cm == 2 && cn == 1) return f(ConvKernel<T, BN, BKB, 2, false, true, 2, 1, RES, TMA>());
    if (cm == 1 && cn == 2) return f(ConvKernel<T, BN, BKB, 2, false, true, 1, 2, RES, TMA>());
    if (cm == 2 && cn == 2) return f(ConvKernel<T, BN, BKB, 2, false, true, 2, 2, RES, TMA>());
  }
  return no_conv_kernel(p);
}
// ... and the epilogue: staged, or (16-bit) the TMA store
template <typename T, int BN, int BKB, bool RES, typename F>
static int conv_kernel_pp(const ConvParams& p, F& f) {
  if (!p.epi_tma) return conv_kernel_pp_shape<T, BN, BKB, RES, false>(p, f);
  if constexpr (sizeof(T) == 2) return conv_kernel_pp_shape<T, BN, BKB, RES, true>(p, f);
  return no_conv_kernel(p);
}

template <typename T, int BN, int BKB, bool DET, typename F>
static int conv_kernel_tile(const ConvParams& p, F& f) {
  constexpr bool b16 = sizeof(T) == 2;
  if (p.pingpong) {
    if constexpr (!DET) {
      if (!p.res_smem) return conv_kernel_pp<T, BN, BKB, false>(p, f);
      // the shared-memory shortcut tile: the 128-column, 128-byte k-block tiles of the 16-bit residual convs
      if constexpr (b16 && BN == 128 && BKB == 128) return conv_kernel_pp<T, BN, BKB, true>(p, f);
    }
    return no_conv_kernel(p);
  }
  // cooperative: one instantiation serves every p.cluster x 1 cluster (CM = 0); 16-bit: 2 and 4 CTAs and one consumer
  // warpgroup as well
  const bool shape = p.cluster_n == 1 && (p.cluster == 1 || (b16 && (p.cluster == 2 || p.cluster == 4)));
  if (!shape || p.res_smem) return no_conv_kernel(p);
  if (p.consumers == 2 && !p.epi_tma) return f(ConvKernel<T, BN, BKB, 2, DET>());
  if constexpr (b16 && !DET) {
    if (p.consumers == 2) return f(ConvKernel<T, BN, BKB, 2, false, false, 0, 1, false, true>());
    if (p.consumers == 1 && !p.epi_tma) return f(ConvKernel<T, BN, BKB, 1>());
  }
  return no_conv_kernel(p);
}

template <typename T, typename F>
static int conv_kernel_type(const ConvParams& p, F& f) {
  const int bn = p.block_n, kb = p.block_kb;
  if (p.det_e) {
    // detection heads with the decode fused in: one n-tile holding all 3 (5 + C) columns, the class count read at run
    // time (conv_select picks the width)
    if (bn == 64 && kb == 128) return conv_kernel_tile<T, 64, 128, true>(p, f);
    if (bn == 128 && kb == 128) return conv_kernel_tile<T, 128, 128, true>(p, f);
    if (bn == 256 && kb == 128) return conv_kernel_tile<T, 256, 128, true>(p, f);
    return no_conv_kernel(p);
  }
  if (bn == 128 && kb == 128) return conv_kernel_tile<T, 128, 128, false>(p, f);
  if (bn == 128 && kb == 64) return conv_kernel_tile<T, 128, 64, false>(p, f);
  if (bn == 64 && kb == 128) return conv_kernel_tile<T, 64, 128, false>(p, f);
  if (bn == 64 && kb == 64) return conv_kernel_tile<T, 64, 64, false>(p, f);
  return no_conv_kernel(p);
}

// The instantiation table: every conv_igemm_kernel that exists is named here and nowhere else.  Calls
// f(ConvKernel<...>()) with the instantiation of the schedule conv_select recorded in p and returns what f returns, or
// YB_ERR_UNSUPPORTED when there is none.  conv_select, the launch, the grid query and yb_conv_schedule's ring depth all
// look kernels up here.
template <typename F>
static int conv_kernel_for(const ConvParams& p, F&& f) {
  if (p.dtype == YB_F16) return conv_kernel_type<__half>(p, f);
  if (p.dtype == YB_BF16) return conv_kernel_type<__nv_bfloat16>(p, f);
  if (p.dtype == YB_E4M3) return conv_kernel_type<__nv_fp8_e4m3>(p, f);
  return no_conv_kernel(p);
}

// the persistent grid of kernel K for p on the current device, and the most clusters of p.cluster CTAs resident at once
template <typename K>
static int conv_kernel_grid(const ConvParams& p, int* grid, int* max_clusters) {
  static DeviceOnce once;
  static ClusterCapacity capacity;
  const void* kern = reinterpret_cast<const void*>(K::kernel);
  int rc = ensure_smem_attr(once, kern, K::C::SMEM_BYTES);
  if (rc) return rc;
  *max_clusters = num_sms();
  if (p.cluster > 1) {
    rc = cluster_capacity(capacity, kern, K::C::THREADS, K::C::SMEM_BYTES, p.cluster, max_clusters);
    if (rc) return rc;
  }
  *grid = conv_grid(p, num_sms(), *max_clusters);
  return YB_OK;
}

// Launch a prepared conv (conv_prepare): the kernel conv_select recorded in l.p, with the maps built for it
int conv_launch(const ConvLaunch& l, cudaStream_t st) {
  const ConvParams& p = l.p;
  return conv_kernel_for(p, [&](auto k) -> int {
    using K = decltype(k);
    int grid = 0, max_clusters = 0;
    const int rc = conv_kernel_grid<K>(p, &grid, &max_clusters);
    if (rc) return rc;
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(K::C::THREADS);
    cfg.dynamicSmemBytes = K::C::SMEM_BYTES;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = p.cluster; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    YB_CUDA(cudaLaunchKernelEx(&cfg, K::kernel, l.tmA, l.tmB, p));
    return YB_OK;
  });
}

int conv_launch_grid(const ConvParams& p, int* grid, int* max_clusters) {
  return conv_kernel_for(p, [&](auto k) -> int { return conv_kernel_grid<decltype(k)>(p, grid, max_clusters); });
}

// bytes of one k-block row: 64 / 32 channels of fp16 / bf16, 128 / 64 channels of e4m3
static int conv_block_kb(int cin, int dtype) { return cin * tm_esize(dtype) % 128 == 0 ? 128 : 64; }

// Shape checks, tiling and kernel variant of one conv: everything conv_prepare decides before it looks at the data
// pointers, down to the conv_igemm_kernel instantiation, which must exist.  The launches, yb_conv_schedule and
// yb_net_layer_schedule all select through here.
int conv_select(const ConvRequest& r, ConvParams* p) {
  memset(p, 0, sizeof(*p));
  const yb_conv_desc* d = &r.d;
  const bool win = r.kh != 0 || r.kw != 0;
  const int det = r.det_e;
  if (det && d->cout != 3 * det) {
    set_error("fused decode: %d output channels are not 3 x (5 + %d classes)", d->cout, det - 5);
    return YB_ERR_UNSUPPORTED;
  }
  // the three anchors of a cell share one n-tile of at most 256 columns: 1 to 80 classes
  YB_REQUIRE(det >= 0 && 3 * det <= 256, "fused decode: the %d columns of %d classes do not fit one 256-column tile "
             "(at most 80 classes; more take forward + predict + nms)", 3 * det, det - 5);
  if (win) {
    YB_REQUIRE(r.kh >= 1 && r.kh <= 2 && r.kw >= 1 && r.kw <= 2 && r.scatter >= 0 && r.scatter <= 4, "conv: bad window");
    YB_REQUIRE(d->stride == 1 && !d->out_fp32 && !d->upsample2x && !r.stats,
               "conv: windows are stride-1, 16-bit, non-upsampled and without statistics");
  }
  YB_REQUIRE(win || d->ksize == 1 || d->ksize == 3, "conv: ksize must be 1 or 3 (got %d)", d->ksize);
  YB_REQUIRE(d->stride == 1 || d->stride == 2, "conv: stride must be 1 or 2 (got %d)", d->stride);
  YB_REQUIRE(!(d->ksize == 1 && d->stride != 1), "conv: 1x1 stride-2 is not on the YOLOv3 path");
  YB_REQUIRE(d->cin % 32 == 0 && d->cin >= 32, "conv: cin must be a multiple of 32 (got %d); use yb_stem_conv_fwd", d->cin);
  YB_REQUIRE(d->dtype == YB_F16 || d->dtype == YB_BF16 || d->dtype == YB_E4M3, "conv: dtype must be f16, bf16 or e4m3");
  const bool e4m3 = d->dtype == YB_E4M3;
  if (e4m3) {
    // 1-byte elements: a k-block row is >= 64 channels, and rows, strides and the 16-channel stores are 16-byte units
    YB_REQUIRE(d->cin % 64 == 0, "conv: e4m3 needs cin %% 64 == 0 (got %d)", d->cin);
    YB_REQUIRE(d->in_ld % 16 == 0 && (d->out_fp32 || d->out_ld % 16 == 0) && d->res_ld % 16 == 0,
               "conv: e4m3 needs in_ld, out_ld and res_ld to be multiples of 16");
    YB_REQUIRE(!win && !r.stats, "conv: e4m3 is a forward inference path (no windows, no statistics)");
    YB_REQUIRE(opt("YB_CONV_EG")[0] != '1' && opt("YB_CONV_MODE")[0] != '2' && opt("YB_CONV_EPI")[0] != 'r',
               "conv: e4m3 runs with two consumer warpgroups, no cluster and the staged epilogue "
               "(YB_CONV_EG, YB_CONV_MODE, YB_CONV_EPI are 16-bit only)");
  }
  YB_REQUIRE(d->h % d->stride == 0 && d->w % d->stride == 0, "conv: h,w must be divisible by stride");
  YB_REQUIRE(d->in_ld >= d->cin && d->in_ld % 8 == 0, "conv: in_ld %d invalid for cin %d", d->in_ld, d->cin);
  const int cout_pad = yb_conv_cout_pad(d->cout);
  if (!d->out_fp32) {
    YB_REQUIRE(d->cout % 32 == 0, "conv: 16-bit output needs cout %% 32 == 0 (got %d)", d->cout);
    YB_REQUIRE(d->out_ld >= d->cout && d->out_ld % 8 == 0, "conv: out_ld %d invalid", d->out_ld);
  } else {
    YB_REQUIRE(d->out_ld >= d->cout, "conv: out_ld %d invalid", d->out_ld);
  }
  const int P = d->h / d->stride, Q = d->w / d->stride;
  const int kh = win ? r.kh : d->ksize, kw = win ? r.kw : d->ksize;
  const int pad = win ? 0 : d->ksize / 2;
  // fused-decode heads: the narrowest wgmma width that holds all 3 E columns (C 1-16: 64, 17-37: 128, 38-80: 256; a
  // 256-column tile over cout_pad = 192 rows of weights, C 38-59, gets its last 64 rows zero-filled by the TMA)
  const int bn = det ? (3 * det <= 64 ? 64 : 3 * det <= 128 ? 128 : 256) : (cout_pad % 128 == 0 ? 128 : 64);
  p->M = d->n * P * Q; p->P = P; p->Q = Q;
  // Kernel variants (testing / A-B switches; the detection heads always take the default):
  //   YB_CONV_EG=1        one consumer warpgroup per CTA (64-row tiles) instead of two (128-row tiles)
  //   YB_CONV_MODE=2cta   cooperative clusters of 2 x 1 CTAs (YB_CONV_MC=1: 4 x 1), multicasting the weight tile
  //   YB_CONV_EPI=reg     accumulators stored straight from registers (not with BN statistics: those sum columns
  //                       over the staging tile)
  //   YB_CONV_EPI=stage|tma  the staged epilogue everywhere | the TMA-store epilogue (epilogue_tma) wherever it can
  //                       run (below); unset: the TMA store in the 16-bit inference plans, staged elsewhere
  //   YB_CONV_PP=0|1      0: the cooperative schedule wherever ping-pong would run; 1: ping-pong wherever the kernel
  //                       allows it (two consumer warpgroups, no cluster, staged epilogue), the 1x1 convs with
  //                       128-column tiles included; unset: the shape rule below
  //   YB_CONV_CTAS=N      persistent grid capped at N CTAs (rounded down to whole clusters, at least one), so that
  //                       small tests give every CTA and warpgroup many work units; the kernel is unchanged
  //   YB_CONV_MCAST=0|2x1|1x2|2x2   ping-pong multicast clusters (below): 0 off everywhere, AxB that shape on every
  //                       16-bit ping-pong launch; unset: the plan rule in inference plans, off elsewhere
  //   YB_CONV_RES=ldg|smem  launches with a residual: ldg, the epilogue reads it from global memory; smem (or unset),
  //                       the ping-pong kernel prefetches it into shared memory where it can (below)
  p->consumers = (!det && opt("YB_CONV_EG")[0] == '1') ? 1 : 2;
  p->cluster = (!det && opt("YB_CONV_MODE")[0] == '2') ? (opt("YB_CONV_MC")[0] == '1' ? 4 : 2) : 1;
  const char* eo = opt("YB_CONV_EPI");
  YB_REQUIRE(eo[0] == '\0' || strcmp(eo, "reg") == 0 || strcmp(eo, "stage") == 0 || strcmp(eo, "tma") == 0,
             "conv: YB_CONV_EPI must be reg, stage or tma (got '%s')", eo);
  p->epi_reg = (!det && !r.stats && eo[0] == 'r') ? 1 : 0;
  p->ctas = opt_int("YB_CONV_CTAS", 0);
  // ping-pong wherever the default variant runs, except
  //  - the fused-decode heads: their 256-column tile does not fit 128 rows per warpgroup in registers;
  //  - 1x1 convs with 128-column tiles: their main loop (cin / 64 k-blocks) is too short to hide one warpgroup's
  //    128 x 128 staged epilogue, and on H100 they measured 2-7 % slower ping-pong than with two warpgroups sharing
  //    the epilogue.  With the TMA-store epilogue ping-pong measured 2-9 % faster on them instead (one clean run of
  //    two, DESIGN.md §5); the rule is kept until that is measured again.  The 1x1 convs with 64-column tiles and
  //    every windowed conv gain from ping-pong.
  const char* pp = opt("YB_CONV_PP");
  const bool pp_shape = pp[0] == '1' || (pp[0] != '0' && (kh * kw > 1 || bn != 128));
  p->pingpong = (!det && p->consumers == 2 && p->cluster == 1 && !p->epi_reg && pp_shape) ? 1 : 0;
  const int block_m = 64 * p->consumers;
  p->num_m_tiles = ceil_div(p->M, block_m);
  p->num_n_tiles = det ? 1 : cout_pad / bn;
  // Ping-pong clusters, CM m-tiles x CN n-tiles (conv_igemm_kernel, DESIGN.md §4): each CTA reads 1/CN of its
  // im2col / activation tile and 1/CM of its weight tile from L2.  The plan rule (16-bit inference plans, forward
  // layers without statistics): 2 x 2 for the windowed convs with an even n-tile count, 2 x 1 for the other windowed
  // convs; the 1x1 convs, whose activation tile comes from HBM once anyway, stay unclustered.  CN = 2 only where the
  // n-tile count is even (a forced 1x2 / 2x2 falls back to 1x1 / 2x1 elsewhere).
  p->cluster_n = 1;
  if (p->pingpong && !e4m3) {
    const char* mc = opt("YB_CONV_MCAST");
    int cm = 1, cn = 1;
    if (mc[0] != '\0' && mc[0] != '0') {
      YB_REQUIRE((mc[0] == '1' || mc[0] == '2') && mc[1] == 'x' && (mc[2] == '1' || mc[2] == '2') && mc[3] == '\0',
                 "conv: YB_CONV_MCAST must be 0, 2x1, 1x2 or 2x2 (got '%s')", mc);
      cm = mc[0] - '0'; cn = mc[2] - '0';
    } else if (mc[0] == '\0' && r.plan_rule && kh * kw > 1) {
      cm = 2; cn = 2;
    }
    if (p->num_n_tiles % 2 != 0) cn = 1;
    p->cluster = cm * cn;
    p->cluster_n = cn;
  }
  // Shortcut prefetch for launches with a residual: the 16-bit ping-pong kernel with 128 x 128 tiles and 64-channel
  // k-blocks, whose epilogue would otherwise wait one global load per 32-column chunk.
  // The 4-stage operand ring it leaves costs nothing measurable at any residual layer of the network (DESIGN.md §5).
  // Not for outputs stored elsewhere than at the residual's own row (2x upsample, dgrad parity scatter).
  const char* ro = opt("YB_CONV_RES");
  YB_REQUIRE(ro[0] == '\0' || strcmp(ro, "ldg") == 0 || strcmp(ro, "smem") == 0,
             "conv: YB_CONV_RES must be ldg or smem (got '%s')", ro);
  p->dtype = d->dtype;
  p->block_n = bn;
  p->block_kb = conv_block_kb(d->cin, d->dtype);
  p->det_e = det;
  p->res_smem = (r.res && p->pingpong && !e4m3 && !det && bn == 128 && p->block_kb == 128 && !r.scatter &&
                 !d->upsample2x && !d->out_fp32 && strcmp(ro, "ldg") != 0) ? 1 : 0;
  // The TMA-store epilogue writes plain 16-bit [M, cout] boxes of 128-row tiles: no statistics (they sum columns over
  // the staging tile), no fp32 or fused-decode head, no 2x upsample or dgrad window (rows scattered elsewhere), no e4m3,
  // and no residual read from global memory (the address arithmetic beside 128 live accumulators spills): a residual
  // only as the shortcut tile above, which the epilogue updates in place.
  p->epi_tma = ((eo[0] == 't' || (eo[0] == '\0' && r.plan_rule)) && !e4m3 && !det && !r.stats && p->consumers == 2 &&
                !d->out_fp32 && !d->upsample2x && !win && (!r.res || p->res_smem)) ? 1 : 0;
  p->cout = d->cout; p->cin = d->cin; p->ksize = d->ksize; p->stride = d->stride; p->pad = pad;
  p->kh = kh; p->kw = kw; p->scatter = r.scatter;
  p->im2col = kh * kw > 1;
  p->out_fp32 = d->out_fp32; p->leaky = d->leaky; p->upsample = d->upsample2x;
  p->res_scale = 1.f; p->out_inv_scale = 1.f;
  return conv_kernel_for(*p, [](auto) -> int { return YB_OK; });
}

// conv_select, then the tensor maps over the data pointers, which are baked into maps and parameters.
int conv_prepare(const ConvRequest& r, const void* x, const void* w_packed, const float* scale, const float* shift,
                 const void* res, void* out, float* stat_sum, float* stat_sqsum, ConvLaunch* l) {
  ConvParams* p = &l->p;
  int rc = conv_select(r, p);
  if (rc) return rc;
  const yb_conv_desc* d = &r.d;
  YB_REQUIRE(x && w_packed && out && (scale == nullptr) == (shift == nullptr), "conv: null pointer");   // scale = shift = NULL: identity
  YB_REQUIRE(((uintptr_t)x & 15) == 0 && ((uintptr_t)w_packed & 15) == 0 && ((uintptr_t)out & 15) == 0 &&
                 ((uintptr_t)res & 15) == 0,
             "conv: pointers must be 16-byte aligned");
  YB_REQUIRE((res != nullptr) == r.res, "conv: a residual pointer is given exactly when the request has a residual");
  if (res) YB_REQUIRE(d->res_ld >= d->cout && d->res_ld % 8 == 0 && !d->out_fp32, "conv: res_ld %d invalid", d->res_ld);
  YB_REQUIRE((stat_sum == nullptr) == (stat_sqsum == nullptr), "conv: stat_sum/stat_sqsum must both be given");
  YB_REQUIRE((stat_sum != nullptr) == r.stats, "conv: statistics pointers are given exactly when the request has them");
  const int cout_pad = yb_conv_cout_pad(d->cout);
  const int bk = p->block_kb / tm_esize(d->dtype);   // channels per k-block
  const int kh = p->kh, kw = p->kw;
  // TMA boxes: this CTA's share of the A tile (1 / cluster_n of its rows) and of the B tile (1 / (cluster / cluster_n))
  const int a_rows = 64 * p->consumers / p->cluster_n;
  const int b_rows = p->block_n / (p->cluster / p->cluster_n);
  p->scale = scale; p->shift = shift;
  p->out = out; p->out_ld = d->out_ld; p->res = res; p->res_ld = d->res_ld;
  p->stat_sum = stat_sum; p->stat_sqsum = stat_sqsum;
  if (p->res_smem) {
    // the shortcut as a [M, cout] matrix of row pitch res_ld: 128-row x 64-channel boxes, rows past M zero-filled
    rc = make_tmap_2d(&p->tmR, res, d->dtype, p->M, d->cout, d->res_ld, 64 * p->consumers, 64, 0);
    if (rc) return rc;
  }
  if (p->epi_tma) {
    // the output (a channel slice of its buffer included) as a [M, cout] matrix of row pitch out_ld: one warp's 16 rows
    // x 64 channels per store, rows >= M and channels >= cout clipped
    rc = make_tmap_2d(&p->tmO, out, d->dtype, p->M, d->cout, d->out_ld, 16, 64, 0);
    if (rc) return rc;
  }
  if (p->im2col) {
    const bool win = r.kh != 0 || r.kw != 0;
    rc = make_tmap_im2col_px(&l->tmA, x, d->dtype, d->n, d->h, d->w, d->cin, d->in_ld, win ? 1 : d->ksize, d->stride,
                             p->pad, bk, a_rows);
  } else {
    rc = make_tmap_2d(&l->tmA, x, d->dtype, (long)d->n * d->h * d->w, d->cin, d->in_ld, a_rows, bk, 0);
  }
  if (rc) return rc;
  return make_tmap_2d(&l->tmB, w_packed, d->dtype, cout_pad, (long)kh * kw * d->cin, (long)kh * kw * d->cin, b_rows, bk,
                      1);
}

int conv_prepare_dgrad_s2(const yb_conv_desc* fwd, const void* dz, int dz_ld, int k_cout, const void* w_dgrad_s2,
                          const void* res, int res_ld, void* dx, int dx_ld, ConvLaunch* l) {
  YB_REQUIRE(fwd && dz && w_dgrad_s2 && dx, "dgrad_s2: null pointer");
  YB_REQUIRE(fwd->ksize == 3 && fwd->stride == 2 && fwd->h % 2 == 0 && fwd->w % 2 == 0, "dgrad_s2: 3x3 stride-2 convs only");
  YB_REQUIRE(k_cout >= fwd->cout && k_cout % 32 == 0 && dz_ld >= k_cout, "dgrad_s2: dz must hold k_cout (multiple of 32) channels");
  ConvRequest r{*fwd};
  yb_conv_desc& d = r.d;
  d.h = fwd->h / 2; d.w = fwd->w / 2; d.cin = k_cout; d.cout = fwd->cin; d.ksize = 1; d.stride = 1;
  d.in_ld = dz_ld; d.out_ld = dx_ld; d.res_ld = res_ld; d.out_fp32 = 0; d.leaky = 0; d.upsample2x = 0;
  r.res = res != nullptr;
  const int cin_pad = yb_conv_cout_pad(fwd->cin);
  for (int c = 0; c < 4; ++c) {
    r.kh = 1 + (c >> 1); r.kw = 1 + (c & 1); r.scatter = 1 + c;
    const uint8_t* w = static_cast<const uint8_t*>(w_dgrad_s2) + dgrad_s2_class_offset(c, cin_pad, k_cout) * 2;
    int rc = conv_prepare(r, dz, w, nullptr, nullptr, res, dx, nullptr, nullptr, &l[c]);
    if (rc) return rc;
  }
  return YB_OK;
}

}  // namespace yb

extern "C" int yb_conv_cout_pad(int cout) { return (cout + 63) / 64 * 64; }

// host-only view of conv_select + conv_grid (tests): the kernel yb_conv2d_fwd (kh = kw = 0) or one parity class of
// yb_conv2d_dgrad_s2 (kh x kw window) would launch with the current options on a device with sm_count SMs
extern "C" int yb_conv_schedule(const yb_conv_desc* d, int kh, int kw, int with_stats, int sm_count,
                                yb_conv_schedule_info* info) {
  YB_REQUIRE(d && info && sm_count > 0, "conv_schedule: bad argument");
  yb::ConvRequest r{*d};
  r.kh = kh; r.kw = kw; r.stats = with_stats != 0;
  yb::ConvParams p, pr;   // the launch without a residual, then pr: with one
  int rc = yb::conv_select(r, &p);
  if (rc) return rc;
  r.res = true;
  rc = yb::conv_select(r, &pr);
  if (rc) return rc;
  auto stages = [](const yb::ConvParams& q, int* s) {
    return yb::conv_kernel_for(q, [&](auto k) -> int { *s = decltype(k)::C::STAGES; return YB_OK; });
  };
  rc = stages(p, &info->stages);
  if (rc) return rc;
  rc = stages(pr, &info->res_stages);
  if (rc) return rc;
  info->res_smem = pr.res_smem;
  info->epi_tma = p.epi_tma;
  info->pingpong = p.pingpong;
  info->consumers = p.consumers;
  info->cluster = p.cluster;
  info->block_m = 64 * p.consumers;
  info->block_n = p.block_n;
  info->block_k = p.block_kb / yb::tm_esize(d->dtype);
  info->num_kb = p.kh * p.kw * d->cin / info->block_k;
  info->num_m_tiles = p.num_m_tiles;
  info->num_n_tiles = p.num_n_tiles;
  info->grid = yb::conv_grid(p, sm_count, 0);
  info->cluster_m = p.cluster / p.cluster_n;
  info->cluster_n = p.cluster_n;
  info->units = yb::conv_units(p);
  return YB_OK;
}

extern "C" int yb_conv2d_fwd(const yb_conv_desc* d, const void* x, const void* w_packed, const float* scale,
                             const float* shift, const void* res, void* out, float* stat_sum, float* stat_sqsum,
                             void* stream) {
  if (!d) { yb::set_error("conv: null descriptor"); return YB_ERR_INVALID_ARGUMENT; }
  yb::ConvRequest r{*d};
  r.stats = stat_sum != nullptr;
  r.res = res != nullptr;
  yb::ConvLaunch l;
  int rc = yb::conv_prepare(r, x, w_packed, scale, shift, res, out, stat_sum, stat_sqsum, &l);
  if (rc) return rc;
  return yb::conv_launch(l, static_cast<cudaStream_t>(stream));
}

extern "C" int yb_conv2d_fwd_e4m3(const yb_conv_desc* d, const void* x, const void* w_packed, const float* scale,
                                  const float* shift, const void* res, float res_scale, void* out, float out_scale,
                                  void* stream) {
  YB_REQUIRE(d && d->dtype == YB_E4M3, "conv_e4m3: descriptor dtype must be YB_E4M3");
  YB_REQUIRE(res_scale > 0.f && out_scale > 0.f && isfinite(res_scale) && isfinite(out_scale),
             "conv_e4m3: scales must be positive and finite");
  yb::ConvRequest r{*d};
  r.res = res != nullptr;
  yb::ConvLaunch l;
  int rc = yb::conv_prepare(r, x, w_packed, scale, shift, res, out, nullptr, nullptr, &l);
  if (rc) return rc;
  l.p.res_scale = res_scale;
  l.p.out_inv_scale = 1.f / out_scale;
  return yb::conv_launch(l, static_cast<cudaStream_t>(stream));
}

extern "C" int yb_conv2d_dgrad_s2(const yb_conv_desc* fwd, const void* dz, int dz_ld, int k_cout, const void* w_dgrad_s2,
                                  const void* res, int res_ld, void* dx, int dx_ld, void* stream) {
  yb::ConvLaunch l[4];
  int rc = yb::conv_prepare_dgrad_s2(fwd, dz, dz_ld, k_cout, w_dgrad_s2, res, res_ld, dx, dx_ld, l);
  for (int c = 0; c < 4 && rc == YB_OK; ++c) rc = yb::conv_launch(l[c], static_cast<cudaStream_t>(stream));
  return rc;
}
