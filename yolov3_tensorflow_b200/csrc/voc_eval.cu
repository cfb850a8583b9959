// PASCAL-VOC evaluation on the device: utils/eval_utils.py voc_eval / voc_ap of the reference (:311-423), run for every
// class over a whole validation set (eval.py:114-137).
//   1. voc_match_kernel    : one CTA per image, its ground truth in shared memory; one warp per (image, class) segment of
//                            the NMS output walks the segment in NMS order (= score descending, stable) and applies the
//                            reference's greedy rule: jmax = first argmax of the IoU over ALL gt boxes of the class, TP iff
//                            ovmax > thr and gt jmax is unused.  Appends one 64-bit record per detection to the pool and
//                            adds npos / nd per class.
//   2. voc_sort_*_kernel   : stable LSD radix sort of the records by (class ascending, score descending); ties keep pool
//                            (insertion) order because every pass is stable.
//   3. voc_ap_kernel       : one CTA per class over its sorted segment: cumulative TP / FP counts, rec and prec in float64,
//                            the reverse running maximum of prec, the area terms where recall changes and the 11-point
//                            maxima; the 11-point sum runs on one thread in the reference's order.
// IoU arithmetic is numpy 2's evaluation of voc_eval's expression: detection coordinates float32, the detection's own
// area in float32 (NEP 50: float32 scalar + Python float stays float32), everything else float64 with the ground truth
// in float64.  All of it is spelled with __f*_rn / __d*_rn so that no FMA contraction changes a rounding.
#include "common.cuh"

namespace yb {

static constexpr int MATCH_THREADS = 256;
static constexpr int SORT_THREADS = 256;                  // == radix (one thread per digit in the scatter prologue)
static constexpr int SORT_WARPS = SORT_THREADS / 32;
static constexpr int SORT_IPT = 16;                       // records per thread
static constexpr int SORT_TILE = SORT_THREADS * SORT_IPT;
static constexpr int SCAN_THREADS = 1024;
static constexpr int AP_THREADS = 512;
static constexpr int AP_IPT = 4;
static constexpr int AP_CHUNK = AP_THREADS * AP_IPT;
static constexpr int VOC_MAX_CLASSES = 65535;             // the class field of a record is 16 bits and C is the sentinel
static constexpr int GT_SMEM_BYTES = 4 * sizeof(double) + sizeof(int) + 1;

typedef unsigned long long u64;

// record: bit 0 TP | bits 1..32 descending-score key | bits 33..48 class (C = detection without a class, sorted last)
__device__ __forceinline__ uint32_t score_desc_key(float f) {
  f = f + 0.0f;                                           // -0 == +0, as numpy compares them
  const uint32_t u = __float_as_uint(f);
  const uint32_t asc = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
  return ~asc;
}
__device__ __forceinline__ u64 make_record(int cls, float score, int tp) {
  return ((u64)(uint32_t)cls << 33) | ((u64)score_desc_key(score) << 1) | (u64)(tp & 1);
}

template <typename T>
struct OpAdd { __device__ __forceinline__ T operator()(T a, T b) const { return a + b; } };
struct OpMaxD { __device__ __forceinline__ double operator()(double a, double b) const { return fmax(a, b); } };

// Block-wide exclusive scan in thread order (NT threads, all of them call it; thread 0 gets `ident`); `total` = the
// reduction over all threads.  s_warp holds NT/32 elements; the function leaves it free for reuse.
template <int NT, typename T, typename Op>
__device__ __forceinline__ T block_excl_scan(T v, T ident, Op op, T* s_warp, T& total) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  T incl = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const T u = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl = op(u, incl);
  }
  T excl = __shfl_up_sync(0xffffffffu, incl, 1);
  if (lane == 0) excl = ident;
  if (lane == 31) s_warp[w] = incl;
  __syncthreads();
  if (w == 0) {
    T x = lane < NT / 32 ? s_warp[lane] : ident;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const T u = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x = op(u, x);
    }
    if (lane < NT / 32) s_warp[lane] = x;
  }
  __syncthreads();
  if (w > 0) excl = op(s_warp[w - 1], excl);
  total = s_warp[NT / 32 - 1];
  __syncthreads();
  return excl;
}
template <int NT, typename T, typename Op>
__device__ __forceinline__ T block_reduce(T v, T ident, Op op, T* s_warp) {
  T total;
  block_excl_scan<NT>(v, ident, op, s_warp, total);
  return total;
}

__device__ __forceinline__ int clamp_count(int k, int cap) { return k < 0 ? 0 : (k > cap ? cap : k); }

// first index in [0, K) whose label is >= c (labels ascending)
__device__ __forceinline__ int lower_bound_label(const int* lb, int K, int c) {
  int lo = 0, hi = K;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (lb[mid] < c) lo = mid + 1; else hi = mid;
  }
  return lo;
}

__global__ void __launch_bounds__(MATCH_THREADS)
voc_match_kernel(const float4* __restrict__ boxes, const float* __restrict__ scores, const int* __restrict__ labels,
                 const int* __restrict__ counts, int cap, const double* __restrict__ gt_boxes,
                 const int* __restrict__ gt_labels, const int* __restrict__ gt_counts, int vmax, int C, double thr,
                 u64* __restrict__ pool, long long pool_offset, long long pool_capacity, u64* __restrict__ class_counts) {
  extern __shared__ __align__(16) uint8_t vm_smem[];
  double* sgt = reinterpret_cast<double*>(vm_smem);                  // [vmax][4]
  int* slab = reinterpret_cast<int*>(sgt + 4 * vmax);                // [vmax]
  uint8_t* sused = reinterpret_cast<uint8_t*>(slab + vmax);          // [vmax]
  __shared__ long long s_red[MATCH_THREADS / 32];
  const int img = blockIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;

  // pool position of this image's first detection: pool_offset + sum of the earlier images' counts
  long long acc = 0;
  for (int i = threadIdx.x; i < img; i += MATCH_THREADS) acc += clamp_count(counts[i], cap);
  const long long base = pool_offset + block_reduce<MATCH_THREADS>(acc, 0ll, OpAdd<long long>(), s_red);

  const int V = clamp_count(gt_counts[img], vmax);
  for (int j = threadIdx.x; j < V; j += MATCH_THREADS) {
    const long long g = (long long)img * vmax + j;
#pragma unroll
    for (int e = 0; e < 4; ++e) sgt[4 * j + e] = gt_boxes[4 * g + e];
    const int l = gt_labels[g];
    slab[j] = l;
    sused[j] = 0;
    if (l >= 0 && l < C) atomicAdd(&class_counts[2 * l], 1ull);     // npos (labels outside [0, C) belong to no class)
  }
  __syncthreads();

  const int K = clamp_count(counts[img], cap);
  const long long o = (long long)img * cap;
  const int* lb = labels + o;
  const float* sc = scores + o;
  const float4* bx = boxes + o;
  for (int k = threadIdx.x; k < K; k += MATCH_THREADS) {
    const int l = lb[k];
    if ((l < 0 || l >= C) && base + k < pool_capacity) pool[base + k] = make_record(C, sc[k], 0);
  }
  for (int c = warp; c < C; c += MATCH_THREADS / 32) {
    const int s = lower_bound_label(lb, K, c);
    const int e = lower_bound_label(lb, K, c + 1);
    if (s == e) continue;
    if (lane == 0) atomicAdd(&class_counts[2 * c + 1], (u64)(e - s));  // nd
    for (int k = s; k < e; ++k) {
      const float4 b = bx[k];
      // (bb[2] - bb[0] + 1.) * (bb[3] - bb[1] + 1.) in float32
      const float da = __fmul_rn(__fadd_rn(__fsub_rn(b.z, b.x), 1.f), __fadd_rn(__fsub_rn(b.w, b.y), 1.f));
      const double bx0 = b.x, by0 = b.y, bx1 = b.z, by1 = b.w;
      double best = -INFINITY;
      int bj = -1;
      for (int j = lane; j < V; j += 32) {
        if (slab[j] != c) continue;
        const double g0 = sgt[4 * j], g1 = sgt[4 * j + 1], g2 = sgt[4 * j + 2], g3 = sgt[4 * j + 3];
        const double iw = fmax(__dadd_rn(__dsub_rn(fmin(g2, bx1), fmax(g0, bx0)), 1.0), 0.0);
        const double ih = fmax(__dadd_rn(__dsub_rn(fmin(g3, by1), fmax(g1, by0)), 1.0), 0.0);
        const double inter = __dmul_rn(iw, ih);
        const double ga = __dmul_rn(__dadd_rn(__dsub_rn(g2, g0), 1.0), __dadd_rn(__dsub_rn(g3, g1), 1.0));
        const double ov = __ddiv_rn(inter, __dsub_rn(__dadd_rn((double)da, ga), inter));
        if (ov > best) { best = ov; bj = j; }                        // first maximum of this lane's boxes
      }
      // (ov descending, index ascending) over the warp: np.argmax's first maximum
#pragma unroll
      for (int sh = 16; sh > 0; sh >>= 1) {
        const double ob = __shfl_xor_sync(0xffffffffu, best, sh);
        const int oj = __shfl_xor_sync(0xffffffffu, bj, sh);
        if (oj >= 0 && (bj < 0 || ob > best || (ob == best && oj < bj))) { best = ob; bj = oj; }
      }
      const int tp = (bj >= 0 && best > thr && !sused[bj]) ? 1 : 0;
      __syncwarp();
      if (lane == 0) {
        if (tp) sused[bj] = 1;
        if (base + k < pool_capacity) pool[base + k] = make_record(c, sc[k], tp);
      }
      __syncwarp();
    }
  }
}

__device__ __forceinline__ int radix_digit(u64 r, int shift) { return (int)((r >> shift) & 255u); }

// per-tile digit counts, digit-major: hist[d * num_tiles + tile]
__global__ void __launch_bounds__(SORT_THREADS)
voc_sort_hist_kernel(const u64* __restrict__ in, long long n, int shift, int num_tiles, int* __restrict__ hist) {
  __shared__ int h[256];
  h[threadIdx.x] = 0;
  __syncthreads();
  const long long t0 = (long long)blockIdx.x * SORT_TILE;
  for (int i = threadIdx.x; i < SORT_TILE; i += SORT_THREADS) {
    const long long p = t0 + i;
    if (p < n) atomicAdd(&h[radix_digit(in[p], shift)], 1);
  }
  __syncthreads();
  hist[(long long)threadIdx.x * num_tiles + blockIdx.x] = h[threadIdx.x];
}

// one CTA per digit: exclusive scan over the tiles in place, the digit's total into totals[d]
__global__ void __launch_bounds__(SCAN_THREADS)
voc_sort_scan_kernel(int* __restrict__ hist, int num_tiles, int* __restrict__ totals) {
  __shared__ int s_w[SCAN_THREADS / 32];
  int* row = hist + (long long)blockIdx.x * num_tiles;
  int carry = 0;
  for (int c0 = 0; c0 < num_tiles; c0 += SCAN_THREADS) {
    const int i = c0 + threadIdx.x;
    const int v = i < num_tiles ? row[i] : 0;
    int tot;
    const int excl = block_excl_scan<SCAN_THREADS>(v, 0, OpAdd<int>(), s_w, tot);
    if (i < num_tiles) row[i] = carry + excl;
    carry += tot;
  }
  if (threadIdx.x == 0) totals[blockIdx.x] = carry;
}

// Stable scatter of one tile: warp w owns a contiguous sub-range and ranks its records chunk by chunk in order
// (match_any groups equal digits); ranks are then offset by the earlier warps' counts, the tile's offset and the digit's base.
__global__ void __launch_bounds__(SORT_THREADS)
voc_sort_scatter_kernel(const u64* __restrict__ in, u64* __restrict__ out, long long n, int shift, int num_tiles,
                        const int* __restrict__ hist, const int* __restrict__ totals) {
  static_assert(SORT_THREADS == 256, "one thread per digit");
  __shared__ int s_cnt[SORT_WARPS][256];
  __shared__ int s_goff[256];
  __shared__ int s_w[SORT_THREADS / 32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, d0 = threadIdx.x;
  const int tot = totals[d0];
  int all;
  s_goff[d0] = block_excl_scan<SORT_THREADS>(tot, 0, OpAdd<int>(), s_w, all) + hist[(long long)d0 * num_tiles + blockIdx.x];
#pragma unroll
  for (int ww = 0; ww < SORT_WARPS; ++ww) s_cnt[ww][d0] = 0;
  __syncthreads();
  const long long t0 = (long long)blockIdx.x * SORT_TILE + (long long)w * (SORT_TILE / SORT_WARPS);
  u64 rec[SORT_IPT];
  int pos[SORT_IPT];
#pragma unroll
  for (int j = 0; j < SORT_IPT; ++j) {
    const long long p = t0 + j * 32 + lane;
    const bool valid = p < n;
    const u64 r = valid ? in[p] : 0ull;
    const int d = valid ? radix_digit(r, shift) : 256;
    const unsigned peers = __match_any_sync(0xffffffffu, d);
    const int rank = __popc(peers & ((1u << lane) - 1u));
    const int b = valid ? s_cnt[w][d] : 0;
    __syncwarp();
    if (valid && rank == 0) s_cnt[w][d] = b + __popc(peers);
    __syncwarp();
    rec[j] = r;
    pos[j] = valid ? b + rank : -1;
  }
  __syncthreads();
  {
    int run = 0;
#pragma unroll
    for (int ww = 0; ww < SORT_WARPS; ++ww) { const int t = s_cnt[ww][d0]; s_cnt[ww][d0] = run; run += t; }
  }
  __syncthreads();
#pragma unroll
  for (int j = 0; j < SORT_IPT; ++j) {
    if (pos[j] >= 0) {
      const int d = radix_digit(rec[j], shift);
      out[(long long)s_goff[d] + s_cnt[w][d] + pos[j]] = rec[j];
    }
  }
}

// One CTA per class over its sorted segment.  Positions p = 0..nd-1 (score descending); the segment is walked from its
// end (q = nd-1-p ascending) so that the envelope max(prec[p..]) and the TP count after p are forward scans in q.
__global__ void __launch_bounds__(AP_THREADS)
voc_ap_kernel(const u64* __restrict__ sorted, const u64* __restrict__ class_counts, int C, int use_07_metric,
              double* __restrict__ out) {
  __shared__ long long s_l[AP_THREADS / 32];
  __shared__ double s_d[AP_THREADS / 32];
  const int c = blockIdx.x;
  long long acc = 0;
  for (int i = threadIdx.x; i < c; i += AP_THREADS) acc += (long long)class_counts[2 * i + 1];
  const long long off = block_reduce<AP_THREADS>(acc, 0ll, OpAdd<long long>(), s_l);
  const long long npos = (long long)class_counts[2 * c], nd = (long long)class_counts[2 * c + 1];
  double* o = out + 5 * (long long)c;
  if (nd == 0) {                                          // voc_eval: 'no box, ignore'
    if (threadIdx.x == 0) { o[0] = 1e-6; o[1] = 1e-6; o[2] = 0.0; o[3] = 0.0; o[4] = 0.0; }
    return;
  }
  const u64* seg = sorted + off;
  long long t = 0;
  for (long long i = threadIdx.x; i < nd; i += AP_THREADS) t += (long long)(seg[i] & 1ull);
  const long long ntp = block_reduce<AP_THREADS>(t, 0ll, OpAdd<long long>(), s_l);
  const double dnpos = (double)npos;

  double area = 0.0;                                      // this thread's share of the area sum
  double m11[11];                                         // max prec over rec >= k/10 (-1: no such position)
#pragma unroll
  for (int k = 0; k < 11; ++k) m11[k] = -1.0;
  long long after = 0;                                    // TPs at positions after the current chunk
  double env_after = 0.0;                                 // max prec after the current chunk (mpre's trailing 0)
  for (long long q0 = 0; q0 < nd; q0 += AP_CHUNK) {
    int tpv[AP_IPT];
    long long s = 0;
#pragma unroll
    for (int j = 0; j < AP_IPT; ++j) {
      const long long q = q0 + (long long)threadIdx.x * AP_IPT + j;
      tpv[j] = q < nd ? (int)(seg[nd - 1 - q] & 1ull) : 0;
      s += tpv[j];
    }
    long long chunk_tp;
    long long run = after + block_excl_scan<AP_THREADS>(s, 0ll, OpAdd<long long>(), s_l, chunk_tp);
    double lmax = 0.0;                                    // prec >= 0, so 0 is the identity of the max
    double prec[AP_IPT], rec[AP_IPT], rprev[AP_IPT];
#pragma unroll
    for (int j = 0; j < AP_IPT; ++j) {
      const long long q = q0 + (long long)threadIdx.x * AP_IPT + j;
      const long long p = nd - 1 - q;
      run += tpv[j];                                      // TPs at positions >= p
      const long long tp = ntp - run + tpv[j];            // cumulative TPs up to p
      prec[j] = q < nd ? __ddiv_rn((double)tp, (double)(p + 1)) : 0.0;   // tp / max(tp + fp, eps), tp + fp = p + 1
      rec[j] = __ddiv_rn((double)tp, dnpos);
      rprev[j] = p == 0 ? 0.0 : __ddiv_rn((double)(tp - tpv[j]), dnpos);
      lmax = fmax(lmax, prec[j]);
    }
    double chunk_max;
    double env = fmax(env_after, block_excl_scan<AP_THREADS>(lmax, 0.0, OpMaxD(), s_d, chunk_max));
#pragma unroll
    for (int j = 0; j < AP_IPT; ++j) {
      const long long q = q0 + (long long)threadIdx.x * AP_IPT + j;
      if (q >= nd) continue;
      env = fmax(env, prec[j]);                           // mpre[p + 1] after np.maximum.accumulate from the right
      if (rec[j] != rprev[j]) area = __dadd_rn(area, __dmul_rn(__dsub_rn(rec[j], rprev[j]), env));
#pragma unroll
      for (int k = 0; k < 11; ++k)
        if (rec[j] >= __dmul_rn((double)k, 0.1)) m11[k] = fmax(m11[k], prec[j]);   // np.arange(0., 1.1, 0.1)[k]
    }
    after += chunk_tp;
    env_after = fmax(env_after, chunk_max);
  }
  area = block_reduce<AP_THREADS>(area, 0.0, OpAdd<double>(), s_d);
#pragma unroll
  for (int k = 0; k < 11; ++k) m11[k] = block_reduce<AP_THREADS>(m11[k], -1.0, OpMaxD(), s_d);
  if (threadIdx.x == 0) {
    const double rec_last = __ddiv_rn((double)ntp, dnpos);
    if (rec_last != 1.0) area = __dadd_rn(area, __dmul_rn(__dsub_rn(1.0, rec_last), 0.0));   // mrec's trailing 1
    double ap07 = 0.0;
    for (int k = 0; k < 11; ++k) ap07 = __dadd_rn(ap07, __ddiv_rn(m11[k] >= 0.0 ? m11[k] : 0.0, 11.0));
    o[0] = (double)npos;
    o[1] = (double)nd;
    o[2] = rec_last;
    o[3] = __ddiv_rn((double)ntp, (double)nd);
    o[4] = use_07_metric ? ap07 : area;
  }
}

}  // namespace yb

using namespace yb;

namespace {

struct VocWs { size_t keys_a, keys_b, hist, totals, total; int num_tiles; };
VocWs voc_layout(long long pool_size) {
  auto al = [](size_t v) { return (v + 255) & ~size_t(255); };
  VocWs w;
  w.num_tiles = (int)((pool_size + SORT_TILE - 1) / SORT_TILE);
  size_t o = 0;
  w.keys_a = o; o = al(o + (size_t)pool_size * 8);
  w.keys_b = o; o = al(o + (size_t)pool_size * 8);
  w.hist = o;   o = al(o + (size_t)w.num_tiles * 256 * 4);
  w.totals = o; o = al(o + 256 * 4);
  w.total = o;
  return w;
}

}  // namespace

extern "C" int yb_voc_match(const float* out_boxes, const float* out_scores, const int32_t* out_labels,
                            const int32_t* counts, int n, int cap, const double* gt_boxes, const int32_t* gt_labels,
                            const int32_t* gt_counts, int vmax, int num_classes, double iou_thresh, uint64_t* pool,
                            long pool_offset, long pool_capacity, uint64_t* class_counts, void* stream) {
  YB_REQUIRE(n >= 0 && n <= 0x7fffffff && cap >= 0, "voc_match: bad shape (n %d, cap %d)", n, cap);
  YB_REQUIRE(vmax >= 0 && vmax <= YB_VOC_MAX_GT, "voc_match: vmax %d outside [0, %d]", vmax, (int)YB_VOC_MAX_GT);
  YB_REQUIRE(num_classes >= 1 && num_classes <= VOC_MAX_CLASSES, "voc_match: num_classes %d outside [1, %d]",
             num_classes, VOC_MAX_CLASSES);
  YB_REQUIRE(pool_offset >= 0 && pool_offset <= pool_capacity, "voc_match: pool offset %ld outside [0, %ld]",
             pool_offset, pool_capacity);
  YB_REQUIRE(class_counts, "voc_match: null pointer");
  if (n == 0) return YB_OK;
  YB_REQUIRE(counts && gt_counts && (cap == 0 || (out_boxes && out_scores && out_labels && pool)) &&
             (vmax == 0 || (gt_boxes && gt_labels)), "voc_match: null pointer");
  YB_REQUIRE(((uintptr_t)out_boxes & 15) == 0, "voc_match: boxes must be 16-byte aligned");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const size_t smem = (size_t)vmax * GT_SMEM_BYTES;      // <= 37 KB at YB_VOC_MAX_GT: no opt-in needed
  voc_match_kernel<<<n, MATCH_THREADS, smem, st>>>(reinterpret_cast<const float4*>(out_boxes), out_scores, out_labels,
                                                   counts, cap, gt_boxes, gt_labels, gt_counts, vmax, num_classes,
                                                   iou_thresh, reinterpret_cast<u64*>(pool), pool_offset, pool_capacity,
                                                   reinterpret_cast<u64*>(class_counts));
  YB_CUDA(cudaGetLastError());
  return YB_OK;
}

extern "C" int yb_voc_ap_workspace_bytes(long pool_size, int num_classes, size_t* bytes) {
  YB_REQUIRE(bytes && pool_size >= 0 && pool_size <= 0x7fffffffL, "voc_ap: bad pool size %ld", pool_size);
  YB_REQUIRE(num_classes >= 1 && num_classes <= VOC_MAX_CLASSES, "voc_ap: num_classes %d outside [1, %d]", num_classes,
             VOC_MAX_CLASSES);
  *bytes = voc_layout(pool_size).total;
  return YB_OK;
}

extern "C" int yb_voc_ap(const uint64_t* pool, long pool_size, const uint64_t* class_counts, int num_classes,
                         int use_07_metric, void* workspace, size_t workspace_bytes, double* out, void* stream) {
  size_t need = 0;
  const int rc = yb_voc_ap_workspace_bytes(pool_size, num_classes, &need);
  if (rc) return rc;
  if (workspace_bytes < need) {
    set_error("voc_ap: workspace too small (%zu < %zu)", workspace_bytes, need);
    return YB_ERR_WORKSPACE;
  }
  YB_REQUIRE(class_counts && out && workspace && (pool_size == 0 || pool), "voc_ap: null pointer");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const VocWs w = voc_layout(pool_size);
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  u64* buf[2] = {reinterpret_cast<u64*>(ws + w.keys_a), reinterpret_cast<u64*>(ws + w.keys_b)};
  int* hist = reinterpret_cast<int*>(ws + w.hist);
  int* totals = reinterpret_cast<int*>(ws + w.totals);
  const u64* src = reinterpret_cast<const u64*>(pool);
  if (pool_size > 0) {
    // digits over bits 1..48 of the record, least significant first: 4 score digits, then 1 or 2 class digits
    const int passes = 4 + (num_classes <= 255 ? 1 : 2);
    for (int p = 0; p < passes; ++p) {
      const int shift = 1 + 8 * p;
      u64* dst = buf[p & 1];
      voc_sort_hist_kernel<<<w.num_tiles, SORT_THREADS, 0, st>>>(src, pool_size, shift, w.num_tiles, hist);
      YB_CUDA(cudaGetLastError());
      voc_sort_scan_kernel<<<256, SCAN_THREADS, 0, st>>>(hist, w.num_tiles, totals);
      YB_CUDA(cudaGetLastError());
      voc_sort_scatter_kernel<<<w.num_tiles, SORT_THREADS, 0, st>>>(src, dst, pool_size, shift, w.num_tiles, hist, totals);
      YB_CUDA(cudaGetLastError());
      src = dst;
    }
  }
  voc_ap_kernel<<<num_classes, AP_THREADS, 0, st>>>(src, reinterpret_cast<const u64*>(class_counts), num_classes,
                                                    use_07_metric ? 1 : 0, out);
  YB_CUDA(cudaGetLastError());
  return YB_OK;
}
