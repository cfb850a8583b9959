// k-means anchors on the device: get_kmeans.py's kmeans / avg_iou of the reference (:32-41, :59-93), bit for bit.
//   1. kmeans_assign_kernel : grid-stride over the boxes, the k clusters in shared memory; d = 1 - IoU per (box, cluster)
//                             and np.argmin over d (first minimum, first NaN wins).  Each block adds its per-cluster
//                             counts and its number of changes against the last assignment to result[k + 1].
//   2. kmeans_hist_kernel /  : np.median of every (cluster, column) by radix select over the float64 bit patterns
//      kmeans_select_kernel    (positive values order as their bits): 8 passes of 8-bit digits, most significant first.
//                             Each pass histograms, in shared memory, the digit of every box whose higher digits equal
//                             a target's prefix; the select kernel then picks each target's digit and remaining rank.
//                             The two targets of a (cluster, column) are ranks (m-1)/2 and m/2; they share one histogram
//                             until their prefixes differ.  The last pass writes the middle value or (lo + hi) * 0.5.
//   3. kmeans_maxiou_kernel, : avg_iou = numpy's pairwise sum of the per-box max IoU, divided by rows.  The sum tree
//      kmeans_leaf_kernel,     depends only on rows: leaves of at most 128 values summed with 8 accumulators, split at
//      kmeans_combine_kernel   n2 = n/2 - (n/2) % 8 above that.  Leaves are summed in parallel (8 lanes per leaf) into
//                             a slot array indexed by tree path; one launch per level combines left + right.
// Everything is float64, spelled with __d*_rn so that no FMA contraction changes a rounding.
#include "common.cuh"

namespace yb {

static constexpr int KM_MAX_K = YB_KMEANS_MAX_K;
static constexpr int ASSIGN_THREADS = 256;
static constexpr int HIST_THREADS = 512;
static constexpr int SELECT_THREADS = 256;                 // one thread per digit value
static constexpr int LEAF_THREADS = 256;                   // 8 lanes per leaf
static constexpr int COMBINE_THREADS = 256;
static constexpr int PW_BLOCK = 128;                       // numpy's PW_BLOCKSIZE

// per (cluster, column) state of the radix select; lo = rank (m-1)/2, hi = rank m/2 of the m values
struct SelState {
  unsigned long long prefix_lo, prefix_hi;                 // digits chosen so far (lower digits zero)
  int rank_lo, rank_hi;                                    // ranks left inside the current prefix
  int m;                                                   // boxes in the cluster
  int diverged;                                            // prefix_lo != prefix_hi: hi has a histogram of its own
};

// np.minimum: NaN if either operand is NaN
__device__ __forceinline__ double np_min(double a, double b) { return (a < b || a != a) ? a : b; }

// 1 - iou(box, cluster) / iou itself, in the reference's operation order
__device__ __forceinline__ double km_iou(double bw, double bh, double ba, double cw, double ch, double ca) {
  const double inter = __dmul_rn(np_min(cw, bw), np_min(ch, bh));
  return __ddiv_rn(inter, __dadd_rn(__dsub_rn(__dadd_rn(ba, ca), inter), 1e-10));
}

__global__ void __launch_bounds__(ASSIGN_THREADS)
kmeans_assign_kernel(const double2* __restrict__ boxes, long long rows, const double* __restrict__ clusters, int k,
                     const int* last, int* assign, int* __restrict__ result) {   // last may be assign itself
  __shared__ double s_cw[KM_MAX_K], s_ch[KM_MAX_K], s_ca[KM_MAX_K];
  __shared__ int s_cnt[KM_MAX_K + 1];                      // counts, then changes
  for (int c = threadIdx.x; c < k; c += ASSIGN_THREADS) {
    const double cw = clusters[2 * c], ch = clusters[2 * c + 1];
    s_cw[c] = cw;
    s_ch[c] = ch;
    s_ca[c] = __dmul_rn(cw, ch);
  }
  for (int c = threadIdx.x; c <= k; c += ASSIGN_THREADS) s_cnt[c] = 0;
  __syncthreads();
  int changes = 0;
  for (long long i = blockIdx.x * (long long)ASSIGN_THREADS + threadIdx.x; i < rows;
       i += (long long)gridDim.x * ASSIGN_THREADS) {
    const double2 b = boxes[i];
    const int prev = last[i];
    const double ba = __dmul_rn(b.x, b.y);
    int best = 0;
    double best_d = __dsub_rn(1.0, km_iou(b.x, b.y, ba, s_cw[0], s_ch[0], s_ca[0]));
    if (best_d == best_d) {
      for (int c = 1; c < k; ++c) {
        const double d = __dsub_rn(1.0, km_iou(b.x, b.y, ba, s_cw[c], s_ch[c], s_ca[c]));
        if (!(d >= best_d)) {                              // d < best_d, or d is the first NaN
          best = c;
          best_d = d;
          if (d != d) break;
        }
      }
    }
    assign[i] = best;
    changes += best != prev;
    atomicAdd(&s_cnt[best], 1);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) changes += __shfl_down_sync(0xffffffffu, changes, o);
  if ((threadIdx.x & 31) == 0 && changes) atomicAdd(&s_cnt[k], changes);
  __syncthreads();
  for (int c = threadIdx.x; c <= k; c += ASSIGN_THREADS)
    if (s_cnt[c]) atomicAdd(&result[c], s_cnt[c]);
}

// digit `pass` (0 = most significant byte) of every box, counted per target whose prefix it matches
__global__ void __launch_bounds__(HIST_THREADS)
kmeans_hist_kernel(const double2* __restrict__ boxes, long long rows, const int* __restrict__ assign, int k, int pass,
                   const SelState* __restrict__ state, int* __restrict__ ghist) {
  extern __shared__ int s_hist[];                          // [2k pairs][lo, hi][256]
  __shared__ unsigned long long s_plo[2 * KM_MAX_K], s_phi[2 * KM_MAX_K];
  __shared__ int s_div[2 * KM_MAX_K];
  const int P = 2 * k;
  for (int j = threadIdx.x; j < P * 512; j += HIST_THREADS) s_hist[j] = 0;
  for (int p = threadIdx.x; p < P; p += HIST_THREADS) {
    s_plo[p] = pass ? state[p].prefix_lo : 0ull;
    s_phi[p] = pass ? state[p].prefix_hi : 0ull;
    s_div[p] = pass ? state[p].diverged : 0;
  }
  __syncthreads();
  const unsigned long long mask = pass ? ~0ull << (64 - 8 * pass) : 0ull;
  const int shift = 56 - 8 * pass;
  for (long long i = blockIdx.x * (long long)HIST_THREADS + threadIdx.x; i < rows;
       i += (long long)gridDim.x * HIST_THREADS) {
    const int c = assign[i];
    if ((unsigned)c >= (unsigned)k) continue;
    const double2 b = boxes[i];
#pragma unroll
    for (int d = 0; d < 2; ++d) {
      const unsigned long long bits = (unsigned long long)__double_as_longlong(d ? b.y : b.x);
      const int p = 2 * c + d;
      const int dig = (int)((bits >> shift) & 255);
      const unsigned long long pre = bits & mask;
      if (pre == s_plo[p]) atomicAdd(&s_hist[p * 512 + dig], 1);
      if (s_div[p] && pre == s_phi[p]) atomicAdd(&s_hist[p * 512 + 256 + dig], 1);
    }
  }
  __syncthreads();
  for (int j = threadIdx.x; j < P * 512; j += HIST_THREADS)
    if (s_hist[j]) atomicAdd(&ghist[j], s_hist[j]);
}

// inclusive scan of one int per thread over SELECT_THREADS threads
__device__ __forceinline__ int select_scan(int v, int* s_warp) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int u = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += u;
  }
  if (lane == 31) s_warp[w] = v;
  __syncthreads();
  int base = 0;
  for (int j = 0; j < w; ++j) base += s_warp[j];
  __syncthreads();
  return v + base;
}

// one block per (cluster, column): pick this pass's digit of both targets from the histogram, zero the histogram for
// the next pass, and after the last pass write the median
__global__ void __launch_bounds__(SELECT_THREADS)
kmeans_select_kernel(const int* __restrict__ counts, int pass, SelState* __restrict__ state, int* __restrict__ ghist,
                     double* __restrict__ clusters_out) {
  __shared__ int s_warp[SELECT_THREADS / 32];
  __shared__ unsigned long long s_plo, s_phi;
  __shared__ int s_rlo, s_rhi;
  const int p = blockIdx.x, t = threadIdx.x;
  SelState st;
  if (pass == 0) {
    const int m = counts[p >> 1];
    st.prefix_lo = st.prefix_hi = 0ull;
    st.m = m;
    st.rank_lo = m > 0 ? (m - 1) / 2 : 0;
    st.rank_hi = m / 2;
    st.diverged = 0;
  } else {
    st = state[p];
  }
  int* h = ghist + p * 512;
  const int h_lo = h[t], h_hi = h[256 + t];
  h[t] = 0;
  h[256 + t] = 0;
  if (t == 0) {                                            // (only kept if counts disagree with the assignment)
    s_plo = st.prefix_lo;
    s_phi = st.prefix_hi;
    s_rlo = s_rhi = 0;
  }
  if (st.m <= 0) {                                         // np.median of no values
    if (t == 0) {
      state[p] = st;
      if (pass == 7) clusters_out[p] = __longlong_as_double(0x7ff8000000000000ll);
    }
    return;
  }
  const int shift = 56 - 8 * pass;
  const int incl_lo = select_scan(h_lo, s_warp);
  const int incl_hi = st.diverged ? select_scan(h_hi, s_warp) : incl_lo;
  const int excl_lo = incl_lo - h_lo;
  const int excl_hi = incl_hi - (st.diverged ? h_hi : h_lo);
  if (excl_lo <= st.rank_lo && st.rank_lo < incl_lo) {
    s_plo = st.prefix_lo | ((unsigned long long)t << shift);
    s_rlo = st.rank_lo - excl_lo;
  }
  if (excl_hi <= st.rank_hi && st.rank_hi < incl_hi) {
    s_phi = st.prefix_hi | ((unsigned long long)t << shift);
    s_rhi = st.rank_hi - excl_hi;
  }
  __syncthreads();
  if (t == 0) {
    st.prefix_lo = s_plo;
    st.prefix_hi = s_phi;
    st.rank_lo = s_rlo;
    st.rank_hi = s_rhi;
    st.diverged = st.prefix_lo != st.prefix_hi;
    state[p] = st;
    if (pass == 7) {
      const double lo = __longlong_as_double((long long)st.prefix_lo);
      const double hi = __longlong_as_double((long long)st.prefix_hi);
      clusters_out[p] = (st.m & 1) ? lo : __dmul_rn(__dadd_rn(lo, hi), 0.5);
    }
  }
}

// ---- avg_iou: numpy's pairwise summation tree over rows values -------------------------------------------------------
// Node at depth `depth` along path `s` (bits most significant first); false if a leaf ends the path earlier, or, with
// `leaf_ok`, if that leaf is not the leftmost slot below it (the slot that holds it).
__device__ __forceinline__ bool pw_node(long long n, int depth, long long s, bool leaf_ok, long long& start,
                                        long long& size) {
  start = 0;
  size = n;
  for (int l = 0; l < depth; ++l) {
    if (size <= PW_BLOCK) return leaf_ok && (s & ((1ll << (depth - l)) - 1)) == 0;
    long long n2 = size / 2;
    n2 -= n2 % 8;
    if ((s >> (depth - 1 - l)) & 1) { start += n2; size -= n2; } else { size = n2; }
  }
  return true;
}

// vals[i] = np.max(iou(boxes[i], clusters)): the first NaN if there is one
__global__ void __launch_bounds__(ASSIGN_THREADS)
kmeans_maxiou_kernel(const double2* __restrict__ boxes, long long rows, const double* __restrict__ clusters, int k,
                     double* __restrict__ vals) {
  __shared__ double s_cw[KM_MAX_K], s_ch[KM_MAX_K], s_ca[KM_MAX_K];
  for (int c = threadIdx.x; c < k; c += ASSIGN_THREADS) {
    const double cw = clusters[2 * c], ch = clusters[2 * c + 1];
    s_cw[c] = cw;
    s_ch[c] = ch;
    s_ca[c] = __dmul_rn(cw, ch);
  }
  __syncthreads();
  for (long long i = blockIdx.x * (long long)ASSIGN_THREADS + threadIdx.x; i < rows;
       i += (long long)gridDim.x * ASSIGN_THREADS) {
    const double2 b = boxes[i];
    const double ba = __dmul_rn(b.x, b.y);
    double best = km_iou(b.x, b.y, ba, s_cw[0], s_ch[0], s_ca[0]);
    for (int c = 1; c < k && best == best; ++c) {
      const double v = km_iou(b.x, b.y, ba, s_cw[c], s_ch[c], s_ca[c]);
      if (!(v <= best)) best = v;
    }
    vals[i] = best;
  }
}

// slots[leaf's leftmost path at depth D] = numpy's sum of the leaf: 8 lanes per leaf, lane j the accumulator r[j]
__global__ void __launch_bounds__(LEAF_THREADS)
kmeans_leaf_kernel(const double* __restrict__ vals, long long rows, int D, double* __restrict__ slots) {
  const long long g = blockIdx.x * (long long)LEAF_THREADS + threadIdx.x;
  const long long s = g >> 3;
  const int j = (int)(g & 7);
  long long start = 0, size = 0;
  const bool valid = s < (1ll << D) && pw_node(rows, D, s, true, start, size);
  const long long body = size >= 8 ? size - size % 8 : 0;     // below 8 values numpy sums in order from 0
  double r = 0.0;                                             // 0 + v == v: every value is >= 0 or NaN
  if (valid)
    for (long long i = j; i < body; i += 8) r = __dadd_rn(r, vals[start + i]);
  // ((r0 + r1) + (r2 + r3)) + ((r4 + r5) + (r6 + r7))
  r = __dadd_rn(r, __shfl_down_sync(0xffffffffu, r, 1, 8));
  r = __dadd_rn(r, __shfl_down_sync(0xffffffffu, r, 2, 8));
  r = __dadd_rn(r, __shfl_down_sync(0xffffffffu, r, 4, 8));
  if (valid && j == 0) {
    for (long long i = body; i < size; ++i) r = __dadd_rn(r, vals[start + i]);
    slots[s] = r;
  }
}

// depth `depth` of the tree: every internal node adds its right child's slot into its own (= its left child's) slot
__global__ void __launch_bounds__(COMBINE_THREADS)
kmeans_combine_kernel(long long rows, int depth, int D, double* __restrict__ slots) {
  const long long s = blockIdx.x * (long long)COMBINE_THREADS + threadIdx.x;
  if (s >= (1ll << depth)) return;
  long long start, size;
  if (!pw_node(rows, depth, s, false, start, size) || size <= PW_BLOCK) return;
  const long long a = s << (D - depth), b = (2 * s + 1) << (D - depth - 1);
  slots[a] = __dadd_rn(slots[a], slots[b]);
}

__global__ void kmeans_mean_kernel(const double* __restrict__ slots, long long rows, double* __restrict__ out) {
  *out = __ddiv_rn(slots[0], (double)rows);
}

}  // namespace yb

using namespace yb;

namespace {

// depth of numpy's pairwise tree over n values (0: one leaf)
int pw_depth(long long n) {
  long long sizes[64];                                     // the sizes of one level span fewer than 40 values
  int ns = 1, D = 0;
  sizes[0] = n;
  for (;;) {
    long long next[64];
    int nn = 0;
    for (int i = 0; i < ns; ++i) {
      if (sizes[i] <= PW_BLOCK) continue;
      long long n2 = sizes[i] / 2;
      n2 -= n2 % 8;
      const long long kids[2] = {n2, sizes[i] - n2};
      for (long long v : kids) {
        bool seen = false;
        for (int j = 0; j < nn; ++j) seen |= next[j] == v;
        if (!seen && nn < 64) next[nn++] = v;
      }
    }
    if (nn == 0) return D;
    ++D;
    for (int i = 0; i < nn; ++i) sizes[i] = next[i];
    ns = nn;
  }
}

struct KmWs { size_t hist, state, vals, slots, total; int depth; };
KmWs km_layout(long long rows, int k) {
  auto al = [](size_t v) { return (v + 255) & ~size_t(255); };
  KmWs w;
  w.depth = pw_depth(rows);
  size_t o = 0;                                            // avg_iou uses [0, hist) only: it does not depend on k
  w.vals = o;  o = al(o + (size_t)rows * sizeof(double));
  w.slots = o; o = al(o + (sizeof(double) << w.depth));
  w.hist = o;  o = al(o + (size_t)k * 2 * 512 * sizeof(int));
  w.state = o; o = al(o + (size_t)k * 2 * sizeof(SelState));
  w.total = o;
  return w;
}

int km_check(const char* what, long long rows, int k) {
  YB_REQUIRE(k >= 1 && k <= KM_MAX_K, "%s: k %d outside [1, %d]", what, k, KM_MAX_K);
  YB_REQUIRE(rows >= k && rows <= 0x7fffffffll, "%s: rows %lld outside [k = %d, 2^31)", what, rows, k);
  return YB_OK;
}

int km_workspace(const char* what, long long rows, int k, const void* ws, size_t ws_bytes) {
  const size_t need = km_layout(rows, k).total;
  if (ws_bytes < need) {
    set_error("%s: workspace too small (%zu < %zu)", what, ws_bytes, need);
    return YB_ERR_WORKSPACE;
  }
  YB_REQUIRE(ws, "%s: null workspace", what);
  return YB_OK;
}

int grid_for(long long rows, int threads, int per_sm) {
  const long long want = (rows + threads - 1) / threads;
  const long long cap = (long long)num_sms() * per_sm;
  return (int)(want < cap ? (want > 0 ? want : 1) : cap);
}

}  // namespace

extern "C" int yb_kmeans_workspace_bytes(long rows, int k, size_t* bytes) {
  YB_REQUIRE(bytes, "kmeans_workspace_bytes: null pointer");
  if (int rc = km_check("kmeans_workspace_bytes", rows, k)) return rc;
  *bytes = km_layout(rows, k).total;
  return YB_OK;
}

extern "C" int yb_kmeans_assign(const double* boxes, long rows, const double* clusters, int k,
                                const int32_t* last_assign, int32_t* assign, int32_t* result, void* workspace,
                                size_t workspace_bytes, void* stream) {
  if (int rc = km_check("kmeans_assign", rows, k)) return rc;
  if (int rc = km_workspace("kmeans_assign", rows, k, workspace, workspace_bytes)) return rc;
  YB_REQUIRE(boxes && clusters && last_assign && assign && result, "kmeans_assign: null pointer");
  YB_REQUIRE(((uintptr_t)boxes & 15) == 0, "kmeans_assign: boxes must be 16-byte aligned");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  YB_CUDA(cudaMemsetAsync(result, 0, (size_t)(k + 1) * sizeof(int32_t), st));
  kmeans_assign_kernel<<<grid_for(rows, ASSIGN_THREADS, 8), ASSIGN_THREADS, 0, st>>>(
      reinterpret_cast<const double2*>(boxes), rows, clusters, k, last_assign, assign, result);
  YB_CUDA(cudaGetLastError());
  return YB_OK;
}

extern "C" int yb_kmeans_median(const double* boxes, long rows, const int32_t* assign, const int32_t* counts, int k,
                                double* clusters_out, void* workspace, size_t workspace_bytes, void* stream) {
  if (int rc = km_check("kmeans_median", rows, k)) return rc;
  if (int rc = km_workspace("kmeans_median", rows, k, workspace, workspace_bytes)) return rc;
  YB_REQUIRE(boxes && assign && counts && clusters_out, "kmeans_median: null pointer");
  YB_REQUIRE(((uintptr_t)boxes & 15) == 0, "kmeans_median: boxes must be 16-byte aligned");
  static DeviceOnce once;
  const int smem = k * 2 * 512 * (int)sizeof(int);          // 128 KB at k = 32
  if (int rc = ensure_smem_attr(once, (const void*)kmeans_hist_kernel, KM_MAX_K * 2 * 512 * (int)sizeof(int)))
    return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const KmWs w = km_layout(rows, k);
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  int* ghist = reinterpret_cast<int*>(ws + w.hist);
  SelState* state = reinterpret_cast<SelState*>(ws + w.state);
  YB_CUDA(cudaMemsetAsync(ghist, 0, (size_t)k * 2 * 512 * sizeof(int), st));
  const int grid = grid_for(rows, HIST_THREADS, k <= 8 ? 4 : (k <= 16 ? 2 : 1));
  for (int pass = 0; pass < 8; ++pass) {
    kmeans_hist_kernel<<<grid, HIST_THREADS, smem, st>>>(reinterpret_cast<const double2*>(boxes), rows, assign, k,
                                                         pass, state, ghist);
    YB_CUDA(cudaGetLastError());
    kmeans_select_kernel<<<2 * k, SELECT_THREADS, 0, st>>>(counts, pass, state, ghist, clusters_out);
    YB_CUDA(cudaGetLastError());
  }
  return YB_OK;
}

extern "C" int yb_kmeans_avg_iou(const double* boxes, long rows, const double* clusters, int k, double* out,
                                 void* workspace, size_t workspace_bytes, void* stream) {
  YB_REQUIRE(k >= 1 && k <= KM_MAX_K, "kmeans_avg_iou: k %d outside [1, %d]", k, KM_MAX_K);
  YB_REQUIRE(rows >= 1 && rows <= 0x7fffffffl, "kmeans_avg_iou: rows %ld outside [1, 2^31)", rows);
  const KmWs w = km_layout(rows, 1);
  if (workspace_bytes < w.hist) {
    set_error("kmeans_avg_iou: workspace too small (%zu < %zu)", workspace_bytes, w.hist);
    return YB_ERR_WORKSPACE;
  }
  YB_REQUIRE(boxes && clusters && out && workspace, "kmeans_avg_iou: null pointer");
  YB_REQUIRE(((uintptr_t)boxes & 15) == 0, "kmeans_avg_iou: boxes must be 16-byte aligned");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  double* vals = reinterpret_cast<double*>(static_cast<uint8_t*>(workspace) + w.vals);
  double* slots = reinterpret_cast<double*>(static_cast<uint8_t*>(workspace) + w.slots);
  kmeans_maxiou_kernel<<<grid_for(rows, ASSIGN_THREADS, 8), ASSIGN_THREADS, 0, st>>>(
      reinterpret_cast<const double2*>(boxes), rows, clusters, k, vals);
  YB_CUDA(cudaGetLastError());
  const long long leaf_threads = 8ll << w.depth;
  kmeans_leaf_kernel<<<(int)((leaf_threads + LEAF_THREADS - 1) / LEAF_THREADS), LEAF_THREADS, 0, st>>>(
      vals, rows, w.depth, slots);
  YB_CUDA(cudaGetLastError());
  for (int depth = w.depth - 1; depth >= 0; --depth) {
    const long long nodes = 1ll << depth;
    kmeans_combine_kernel<<<(int)((nodes + COMBINE_THREADS - 1) / COMBINE_THREADS), COMBINE_THREADS, 0, st>>>(
        rows, depth, w.depth, slots);
    YB_CUDA(cudaGetLastError());
  }
  kmeans_mean_kernel<<<1, 1, 0, st>>>(slots, rows, out);
  YB_CUDA(cudaGetLastError());
  return YB_OK;
}
