// Batched baseline JPEG decode (replaces cv2.imread at utils/data_utils.py:130 and test_single_image.py:38): BGR
// pixels equal to cv2.imread of OpenCV 4.13 / libjpeg-turbo 3.1, written into the PackedImages layout.
//
// Host: parse the markers up to SOS, build the Huffman decode tables and pack descriptors, tables and the compressed
// bytes of every image into one blob (the batch's one H2D copy).  Device, one launch per stage for the whole batch:
//   1. jpeg_destuff      one CTA per image: find EOI, drop the 00 after FF, split at RST markers; every restart
//                        segment starts on a subsequence boundary of the destuffed stream.
//   2. jpeg_huff_sync    Weissenberger & Schmidt's self-synchronising decode: each thread decodes one subsequence
//                        from a guessed state; threads of a CTA adopt their left neighbour's exit state and decode
//                        again until no start changes; the CTA's first thread takes the exit of the CTA before it
//                        (decoupled look-back in ticket order).  Then a segmented scan of block counts.
//   3. jpeg_huff_decode  re-decodes every subsequence from its synchronised start and scatters the coefficients.
//   4. jpeg_dc           DC differences -> DC values, per component, restarting at each segment.
//   5. jpeg_idct         dequantise + ISLOW IDCT (jidctint.c), saturated as the SIMD path cv2 runs does.
//   6. jpeg_color        fancy upsampling (jdsample.c), YCbCr -> BGR (jdcolor.c), EXIF orientation, store.
#include <limits.h>
#include <string.h>

#include <vector>

#include "common.cuh"

namespace yb {
namespace {

constexpr uint32_t kMagic = 0x4a504231;   // "JPB1"
constexpr int kChunk = 128;               // subsequences per sync CTA
constexpr int kDestuffThreads = 512;
constexpr int kDcThreads = 1024;

__constant__ uint8_t c_zigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,
                                     12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28,
                                     35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
                                     58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
const uint8_t h_zigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                              41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                              30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

struct HuffTab {
  uint16_t fast[512];   // next 9 bits -> (length << 8) | symbol; 0: the code is longer than 9 bits (or invalid)
  int32_t maxcode[18];  // largest code of each length, -1 when there is none
  int32_t valoff[18];   // vals index of a code of length l = code + valoff[l]
  uint8_t vals[256];
};

struct Img {
  int64_t data_off, data_len;     // blob: entropy-coded bytes (SOS end .. end of file)
  int64_t tab_off[3][2];          // blob: DC / AC HuffTab of each component
  int64_t stream_off;             // workspace stream region: destuffed bits, 16-byte aligned
  int64_t sub_base, seg_base;     // first subsequence / segment record of the image
  int64_t coef_off;               // first block (64 int16) of the image in the coefficient region
  int64_t plane_off[3];           // component planes (uint8, MCU-padded) in the plane region
  int64_t pix_off;                // PackedImages pixel offset
  int32_t chunk_base, nsub, nseg, ri, total_mcus, mcus_x, bpm, ncomp;
  int32_t H, W, out_h, out_w, orient, hmax, vmax, pad0;
  int32_t ch[3], cv[3], pw[3], dw[3], dh[3];   // sampling, plane width (blocks), downsampled size
  int8_t blk_comp[8], blk_x[8], blk_y[8];
  uint16_t q[3][64];                            // natural order
};

struct Batch {
  uint32_t magic;
  int32_t n, sub_bits, nchunks;
  int64_t ws_rec, ws_seg, ws_sub, ws_stream, ws_coef, ws_planes, ws_bytes;
  int64_t max_blocks, max_pixels, pixel_bytes;
};

static inline int64_t align16(int64_t v) { return (v + 15) & ~int64_t(15); }

// ---------------------------------------------------------------------------------------------------------------
// host: header parse
// ---------------------------------------------------------------------------------------------------------------
struct Parsed {
  int H = 0, W = 0, nf = 0, ri = 0, orient = 1, mode = 0;
  int id[3], h[3], v[3], tq[3], td[3], ta[3];
  bool have_q[4] = {false, false, false, false};
  uint16_t q[4][64];
  bool have_h[2][4] = {{false, false, false, false}, {false, false, false, false}};
  uint8_t bits[2][4][16];
  uint8_t vals[2][4][256];
  size_t scan_start = 0;
};

static int u16be(const uint8_t* p) { return p[0] << 8 | p[1]; }

#define JREJECT(...) do { set_error(__VA_ARGS__); return YB_ERR_UNSUPPORTED; } while (0)
#define JINVALID(...) do { set_error(__VA_ARGS__); return YB_ERR_INVALID_ARGUMENT; } while (0)

// OpenCV's reading of an APP1 Exif block: tag 0x0112 of IFD0 as a SHORT; a value outside 1..8 means 1.
static int exif_orientation(const uint8_t* s, size_t n) {
  if (n < 14 || memcmp(s, "Exif\0\0", 6) != 0) return 0;
  const uint8_t* t = s + 6;
  n -= 6;
  bool le;
  if (t[0] == 'I' && t[1] == 'I') le = true;
  else if (t[0] == 'M' && t[1] == 'M') le = false;
  else return 1;
  auto r16 = [&](size_t o) { return le ? (t[o] | t[o + 1] << 8) : (t[o] << 8 | t[o + 1]); };
  auto r32 = [&](size_t o) {
    return le ? (uint32_t)t[o] | (uint32_t)t[o + 1] << 8 | (uint32_t)t[o + 2] << 16 | (uint32_t)t[o + 3] << 24
              : (uint32_t)t[o] << 24 | (uint32_t)t[o + 1] << 16 | (uint32_t)t[o + 2] << 8 | (uint32_t)t[o + 3];
  };
  if (n < 8) return 1;
  size_t ifd = r32(4);
  if (ifd + 2 > n) return 1;
  int cnt = r16(ifd);
  for (int e = 0; e < cnt; ++e) {
    size_t o = ifd + 2 + 12 * (size_t)e;
    if (o + 12 > n) break;
    if (r16(o) == 0x0112) {
      int v = r16(o + 8);
      return v >= 1 && v <= 8 ? v : 1;
    }
  }
  return 1;
}

static int parse(const uint8_t* b, size_t n, Parsed& P) {
  YB_REQUIRE(b != nullptr, "jpeg: null data");
  if (n < 4 || b[0] != 0xFF || b[1] != 0xD8) JINVALID("not a JPEG file (no SOI)");
  size_t p = 2;
  bool sof = false, jfif = false;
  int adobe = -1, orient = 0;
  for (;;) {
    if (p >= n || b[p] != 0xFF) JINVALID("marker expected at byte %zu", p);
    while (p < n && b[p] == 0xFF) ++p;
    if (p >= n) JINVALID("truncated header");
    const int m = b[p++];
    if (m == 0xD8 || m == 0x01 || (m >= 0xD0 && m <= 0xD7)) continue;
    if (m == 0xD9) JINVALID("EOI before SOS");
    if (p + 2 > n) JINVALID("truncated header");
    const size_t ln = u16be(b + p);
    if (ln < 2 || p + ln > n) JINVALID("truncated header");
    const uint8_t* s = b + p + 2;
    const size_t sl = ln - 2;
    p += ln;
    if (m == 0xC0 || m == 0xC1) {
      if (sof) JINVALID("second SOF");
      if (sl < 6) JINVALID("bad SOF");
      if (s[0] != 8) JREJECT("%d-bit samples", s[0]);
      P.H = u16be(s + 1);
      P.W = u16be(s + 3);
      P.nf = s[5];
      P.mode = m - 0xC0;
      if (P.H == 0) JREJECT("DNL (height 0 in SOF)");
      if (P.W == 0) JINVALID("width 0");
      if (P.nf == 4) JREJECT("4 components (CMYK / YCCK)");
      if (P.nf != 1 && P.nf != 3) JREJECT("%d components", P.nf);
      if (sl < 6 + 3 * (size_t)P.nf) JINVALID("bad SOF");
      for (int i = 0; i < P.nf; ++i) {
        P.id[i] = s[6 + 3 * i];
        P.h[i] = s[7 + 3 * i] >> 4;
        P.v[i] = s[7 + 3 * i] & 15;
        P.tq[i] = s[8 + 3 * i];
        if (P.tq[i] > 3) JINVALID("bad SOF");
      }
      sof = true;
    } else if (m == 0xC2 || m == 0xC6 || m == 0xCA || m == 0xCE) {
      JREJECT("progressive JPEG");
    } else if (m == 0xC3 || m == 0xC7 || m == 0xCB || m == 0xCF) {
      JREJECT("lossless JPEG");
    } else if (m == 0xC5 || m == 0xDE) {
      JREJECT("hierarchical JPEG");
    } else if (m == 0xC9 || m == 0xCC || m == 0xCD) {
      JREJECT("arithmetic coding");
    } else if (m == 0xC4) {
      size_t o = 0;
      while (o < sl) {
        const int tc = s[o] >> 4, th = s[o] & 15;
        if (tc > 1 || th > 3 || o + 17 > sl) JINVALID("bad DHT");
        int nv = 0;
        for (int l = 0; l < 16; ++l) nv += s[o + 1 + l];
        if (nv > 256 || o + 17 + nv > sl) JINVALID("bad DHT");
        memcpy(P.bits[tc][th], s + o + 1, 16);
        memcpy(P.vals[tc][th], s + o + 17, nv);
        P.have_h[tc][th] = true;
        o += 17 + nv;
      }
    } else if (m == 0xDB) {
      size_t o = 0;
      while (o < sl) {
        const int pq = s[o] >> 4, tq = s[o] & 15;
        if (pq > 1 || tq > 3 || o + 1 + 64 * (pq + 1) > sl) JINVALID("bad DQT");
        for (int i = 0; i < 64; ++i)
          P.q[tq][h_zigzag[i]] = pq ? (uint16_t)u16be(s + o + 1 + 2 * i) : s[o + 1 + i];
        P.have_q[tq] = true;
        o += 1 + 64 * (pq + 1);
      }
    } else if (m == 0xDD) {
      if (sl < 2) JINVALID("bad DRI");
      P.ri = u16be(s);
    } else if (m == 0xE0) {
      if (sl >= 5 && memcmp(s, "JFIF\0", 5) == 0) jfif = true;
    } else if (m == 0xE1) {
      if (orient == 0) orient = exif_orientation(s, sl);
    } else if (m == 0xEE) {
      if (sl >= 12 && memcmp(s, "Adobe", 5) == 0) adobe = s[11];
    } else if (m == 0xDA) {
      if (!sof) JINVALID("SOS before SOF");
      if (sl < 1) JINVALID("bad SOS");
      const int ns = s[0];
      if (ns != P.nf) JREJECT("several scans (non-interleaved)");
      if (sl < 4 + 2 * (size_t)ns) JINVALID("bad SOS");
      bool seen[3] = {false, false, false};
      for (int i = 0; i < ns; ++i) {
        int c = -1;
        for (int j = 0; j < P.nf; ++j)
          if (P.id[j] == s[1 + 2 * i]) c = (c < 0 ? j : -2);
        if (c < 0 || seen[c]) JINVALID("SOS names an unknown component");
        if (c != i) JREJECT("SOS lists the components in another order than SOF");
        seen[c] = true;
        P.td[c] = s[2 + 2 * i] >> 4;
        P.ta[c] = s[2 + 2 * i] & 15;
        if (P.td[c] > 3 || P.ta[c] > 3) JINVALID("bad SOS");
      }
      if (s[1 + 2 * ns] != 0 || s[2 + 2 * ns] != 63 || s[3 + 2 * ns] != 0)
        JREJECT("spectral selection / successive approximation");
      P.scan_start = p;
      break;
    }
  }
  if (P.nf == 3) {
    if (adobe == 0) JREJECT("RGB JPEG (Adobe transform 0)");
    if (adobe < 0 && !jfif && P.id[0] == 'R' && P.id[1] == 'G' && P.id[2] == 'B') JREJECT("RGB JPEG (component ids R, G, B)");
    const bool luma_ok = (P.h[0] == 1 || P.h[0] == 2) && (P.v[0] == 1 || P.v[0] == 2);
    if (!luma_ok || P.h[1] != 1 || P.v[1] != 1 || P.h[2] != 1 || P.v[2] != 1)
      JREJECT("sampling factors %dx%d,%dx%d,%dx%d", P.h[0], P.v[0], P.h[1], P.v[1], P.h[2], P.v[2]);
  } else if (P.h[0] < 1 || P.h[0] > 4 || P.v[0] < 1 || P.v[0] > 4) {
    JINVALID("bad sampling factors");
  }
  for (int c = 0; c < P.nf; ++c) {
    if (!P.have_q[P.tq[c]]) JINVALID("quantisation table %d missing", P.tq[c]);
    if (!P.have_h[0][P.td[c]]) JINVALID("DC Huffman table %d missing", P.td[c]);
    if (!P.have_h[1][P.ta[c]]) JINVALID("AC Huffman table %d missing", P.ta[c]);
  }
  P.orient = orient ? orient : 1;
  return YB_OK;
}

// canonical code assignment (jdhuff.c jpeg_make_d_derived_tbl); an over-full table is invalid
static int build_table(const uint8_t* bits, const uint8_t* vals, HuffTab& t) {
  memset(&t, 0, sizeof(t));
  int code = 0, k = 0;
  for (int l = 1; l <= 16; ++l) {
    t.valoff[l] = k - code;
    for (int i = 0; i < bits[l - 1]; ++i, ++code, ++k) {
      if (l <= 9)
        for (int f = code << (9 - l); f < (code + 1) << (9 - l); ++f) t.fast[f] = (uint16_t)(l << 8 | vals[k]);
    }
    t.maxcode[l] = bits[l - 1] ? code - 1 : -1;
    if (code > (1 << l)) JINVALID("bad Huffman table");
    code <<= 1;
  }
  t.maxcode[17] = 0x7fffffff;
  memcpy(t.vals, vals, k);
  return YB_OK;
}

struct Layout {   // everything pack derives from one header
  Parsed P;
  int bpm, mcus_x, mcus_y, hmax, vmax, ntab;
  int pw[3], ph[3], dw[3], dh[3];
};

static int layout(const uint8_t* data, size_t bytes, Layout& L) {
  int rc = parse(data, bytes, L.P);
  if (rc) return rc;
  const Parsed& P = L.P;
  for (int c = 0; c < P.nf; ++c)
    for (int k = 0; k < 2; ++k) {
      const int id = k ? P.ta[c] : P.td[c];
      HuffTab t;
      if (build_table(P.bits[k][id], P.vals[k][id], t)) return YB_ERR_INVALID_ARGUMENT;
      int nv = 0;
      for (int l = 0; l < 16; ++l) nv += P.bits[k][id][l];
      for (int v = 0; k == 0 && v < nv; ++v)   // jdhuff.c: a DC symbol is a bit count, 0..15
        if (P.vals[0][id][v] > 15) JINVALID("bad DC Huffman table");
    }
  if (P.nf == 1) {
    L.hmax = L.vmax = 1;
    L.mcus_x = (P.W + 7) / 8;
    L.mcus_y = (P.H + 7) / 8;
    L.bpm = 1;
    L.pw[0] = L.mcus_x;
    L.ph[0] = L.mcus_y;
    L.dw[0] = P.W;
    L.dh[0] = P.H;
  } else {
    L.hmax = P.h[0];
    L.vmax = P.v[0];
    L.mcus_x = (P.W + 8 * L.hmax - 1) / (8 * L.hmax);
    L.mcus_y = (P.H + 8 * L.vmax - 1) / (8 * L.vmax);
    L.bpm = P.h[0] * P.v[0] + 2;
    for (int c = 0; c < 3; ++c) {
      L.pw[c] = L.mcus_x * P.h[c];
      L.ph[c] = L.mcus_y * P.v[c];
      L.dw[c] = (P.W * P.h[c] + L.hmax - 1) / L.hmax;
      L.dh[c] = (P.H * P.v[c] + L.vmax - 1) / L.vmax;
    }
  }
  return YB_OK;
}

static int sub_bits_option() { return opt_int("YB_JPEG_SUBSEQ_BITS", 512); }

}  // namespace

// ---------------------------------------------------------------------------------------------------------------
// device
// ---------------------------------------------------------------------------------------------------------------
namespace {

__device__ __forceinline__ uint32_t bswap(uint32_t v) { return __byte_perm(v, 0, 0x0123); }

// 32 bits of the stream starting at bit `pos` (MSB first)
__device__ __forceinline__ uint32_t peek32(const uint32_t* w, uint32_t pos) {
  const uint32_t i = pos >> 5, s = pos & 31;
  const uint64_t v = (uint64_t)bswap(__ldg(w + i)) << 32 | bswap(__ldg(w + i + 1));
  return (uint32_t)((v << s) >> 32);
}

// -> (length << 8) | symbol, or 0 for a code no table holds
__device__ __forceinline__ uint32_t huff(const HuffTab* t, uint32_t bits) {
  const uint32_t e = __ldg(&t->fast[bits >> 23]);
  if (e) return e;
  for (int l = 10; l <= 16; ++l) {
    const int code = (int)(bits >> (32 - l));
    if (code <= __ldg(&t->maxcode[l])) return (uint32_t)l << 8 | __ldg(&t->vals[code + __ldg(&t->valoff[l])]);
  }
  return 0;
}

__device__ __forceinline__ int extend(uint32_t v, int s) { return v < (1u << (s - 1)) ? (int)v - (1 << s) + 1 : (int)v; }

struct State { uint32_t pos, bk; };   // bit position, (block in MCU << 8) | coefficient index k
constexpr uint32_t kErrPos = 0xffffffffu;

__device__ __forceinline__ const HuffTab* table(const uint8_t* blob, const Img& im, int comp, int ac) {
  return reinterpret_cast<const HuffTab*>(blob + im.tab_off[comp][ac]);
}

// Decode codewords from s while s.pos < end.  Returns the number of blocks completed.  WRITE: scatter the
// coefficients of block `first_idx + completed` (DC as a difference) while that index is below `expected`, and
// report errors in those blocks through *err.  An undecodable code ends the walk with s.pos = kErrPos.
template <bool WRITE>
__device__ __forceinline__ int walk(const uint8_t* blob, const Img& im, const uint32_t* words, State& s, uint32_t end, uint32_t first_idx,
                    uint32_t expected, uint32_t seg_end, int16_t* coef, int& err) {
  int done = 0;
  uint32_t pos = s.pos, blk = s.bk >> 8, k = s.bk & 255;
  while (pos < end) {
    const int comp = im.blk_comp[blk];
    const uint32_t bits = peek32(words, pos);
    const uint32_t idx = first_idx + done;
    if (k == 0) {
      const uint32_t e = huff(table(blob, im, comp, 0), bits);
      if (!e) {
        if (WRITE && idx < expected) err |= YB_JPEG_BAD_CODE;
        pos = kErrPos;
        break;
      }
      const int len = e >> 8, t = e & 15;
      const int v = t ? extend((bits << len) >> (32 - t), t) : 0;
      if (WRITE && idx < expected) coef[(size_t)idx * 64] = (int16_t)v;
      pos += len + t;
      k = 1;
    } else {
      const uint32_t e = huff(table(blob, im, comp, 1), bits);
      if (!e) {
        if (WRITE && idx < expected) err |= YB_JPEG_BAD_CODE;
        pos = kErrPos;
        break;
      }
      const int len = e >> 8, r = (e >> 4) & 15, sz = e & 15;
      pos += len;
      if (sz) {
        k += r;
        if (k > 63) {
          if (WRITE && idx < expected) err |= YB_JPEG_BAD_INDEX;
          pos = kErrPos;
          break;
        }
        if (WRITE && idx < expected) coef[(size_t)idx * 64 + c_zigzag[k]] = (int16_t)extend((bits << len) >> (32 - sz), sz);
        pos += sz;
        ++k;
      } else {
        k = r == 15 ? k + 16 : 64;
      }
    }
    if (k >= 64) {
      if (WRITE && idx + 1 == expected && pos > seg_end) err |= YB_JPEG_TRUNCATED;
      k = 0;
      blk = blk + 1 == (uint32_t)im.bpm ? 0 : blk + 1;
      ++done;
    }
  }
  s.pos = pos;
  s.bk = blk << 8 | k;
  return done;
}

__device__ __forceinline__ int find_image(const int32_t* base, int n, int key) {   // last i with base[i] <= key
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (base[mid] <= key) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// per image of the batch: chunk_base copy lives in the blob right after Img[n]
__device__ __forceinline__ const Img* imgs_of(const uint8_t* blob) { return reinterpret_cast<const Img*>(blob + sizeof(Batch)); }
__device__ __forceinline__ const int32_t* chunk_bases(const uint8_t* blob, int n) {
  return reinterpret_cast<const int32_t*>(blob + sizeof(Batch) + sizeof(Img) * (size_t)n);
}

// segment record: start subsequence, length in bits, first destuffed byte index (scratch)
struct Seg { uint32_t start_sub, len_bits, first_emit, pad; };
// subsequence record: synchronised start state and the index of its first block within the segment
struct Sub { uint32_t pos, bk, base, pad; };
// look-back record of a sync CTA
struct Rec { uint32_t pos, bk, count, flag; };

template <typename T>
__device__ __forceinline__ T block_excl_scan(T v, T* smem, T& total) {   // blockDim.x <= 1024, multiple of 32
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  T x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const T y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  __syncthreads();
  if (lane == 31) smem[wid] = x;
  __syncthreads();
  if (wid == 0) {
    T w = lane < nw ? smem[lane] : T(0);
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const T y = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= o) w += y;
    }
    if (lane < nw) smem[lane] = w;
  }
  __syncthreads();
  total = smem[nw - 1];
  return x - v + (wid ? smem[wid - 1] : T(0));
}

// ---- 1. destuff + segment ----
__global__ void __launch_bounds__(kDestuffThreads) jpeg_destuff(const uint8_t* __restrict__ blob, uint8_t* ws,
                                                               int32_t* status) {
  const Batch& B = *reinterpret_cast<const Batch*>(blob);
  const Img& im = imgs_of(blob)[blockIdx.x];
  const uint8_t* d = blob + im.data_off;
  const int64_t n = im.data_len;
  Seg* seg = reinterpret_cast<Seg*>(ws + B.ws_seg) + im.seg_base;
  uint8_t* out = ws + B.ws_stream + im.stream_off;
  const int S = B.sub_bits;
  __shared__ long long s_end;
  __shared__ int s_code;
  __shared__ long long s_scan[32];
  __shared__ long long s_carry[2];
  __shared__ long long s_last_end;   // destuffed index of the first RST past the last segment
  if (threadIdx.x == 0) { s_end = n; s_carry[0] = s_carry[1] = 0; s_last_end = LLONG_MAX; }
  __syncthreads();
  // end of the entropy data: the first FF followed by a byte that is not 00, FF or RSTn
  for (int64_t i = threadIdx.x; i + 1 < n; i += blockDim.x) {
    if (d[i] == 0xFF) {
      const uint8_t c = d[i + 1];
      if (c != 0 && c != 0xFF && (c < 0xD0 || c > 0xD7)) atomicMin(&s_end, (long long)i);
    }
  }
  __syncthreads();
  const int64_t end = s_end;
  if (threadIdx.x == 0) {
    s_code = end < n ? d[end + 1] : 0xD9;
    if (s_code != 0xD9) atomicOr(&status[blockIdx.x], YB_JPEG_BAD_MARKER);
  }
  // byte i is kept unless it follows an FF; an FF is kept when 00 follows it; FF RSTn splits the segments
  auto keep = [&](int64_t i) { return d[i] == 0xFF ? (i + 1 < n && d[i + 1] == 0) : !(i > 0 && d[i - 1] == 0xFF); };
  auto rst = [&](int64_t i) { return d[i] == 0xFF && i + 1 < n && d[i + 1] >= 0xD0 && d[i + 1] <= 0xD7; };
  constexpr int V = 4;
  const int64_t tile = (int64_t)V * blockDim.x;
  // pass 1: the destuffed index at which each segment starts
  for (int64_t t0 = 0; t0 < end; t0 += tile) {
    const int64_t i0 = t0 + (int64_t)V * threadIdx.x;
    long long ke = 0, kr = 0;
    for (int j = 0; j < V; ++j)
      if (i0 + j < end) { ke += keep(i0 + j); kr += rst(i0 + j); }
    long long te, tr;
    const long long pe = block_excl_scan(ke, s_scan, te);
    const long long pr = block_excl_scan(kr, s_scan, tr);
    long long e = s_carry[0] + pe, r = s_carry[1] + pr;
    for (int j = 0; j < V; ++j) {
      const int64_t i = i0 + j;
      if (i >= end) break;
      if (rst(i)) {
        if (d[i + 1] != 0xD0 + (r & 7) || r + 1 >= im.nseg) atomicOr(&status[blockIdx.x], YB_JPEG_BAD_RST);
        if (r + 1 < im.nseg) seg[r + 1].first_emit = (uint32_t)e;
        if (r + 1 == im.nseg) s_last_end = e;
        ++r;
      }
      e += keep(i);
    }
    __syncthreads();
    if (threadIdx.x == 0) { s_carry[0] += te; s_carry[1] += tr; }
    __syncthreads();
  }
  const long long total_e = s_carry[0], total_r = s_carry[1];
  const int nseen = (int)min((long long)im.nseg, s_carry[1] + 1);
  if (threadIdx.x == 0 && nseen < im.nseg) atomicOr(&status[blockIdx.x], YB_JPEG_TRUNCATED);
  __syncthreads();
  // pass 2: segment g starts at subsequence sum over g' < g of ceil(len(g') / S)
  long long carry = 0;
  for (int g0 = 0; g0 < im.nseg; g0 += blockDim.x) {
    const int g = g0 + threadIdx.x;
    uint32_t len = 0;
    if (g < nseen) {
      const long long a = seg[g].first_emit, b = g + 1 < nseen ? (long long)seg[g + 1].first_emit : min(total_e, s_last_end);
      len = (uint32_t)((b - a) * 8);
      if (len == 0) atomicOr(&status[blockIdx.x], YB_JPEG_TRUNCATED);
    }
    long long tot;
    const long long pre = block_excl_scan((long long)((len + S - 1) / S), s_scan, tot);
    if (g < im.nseg) {
      seg[g].start_sub = g < nseen ? (uint32_t)(carry + pre) : 0xffffffffu;
      seg[g].len_bits = len;
    }
    carry += tot;
  }
  __threadfence_block();
  __syncthreads();
  // pass 3: scatter the kept bytes
  for (int64_t t0 = 0; t0 < end; t0 += tile) {
    const int64_t i0 = t0 + (int64_t)V * threadIdx.x;
    long long ke = 0, kr = 0;
    for (int j = 0; j < V; ++j)
      if (i0 + j < end) { ke += keep(i0 + j); kr += rst(i0 + j); }
    long long te, tr;
    const long long pe = block_excl_scan(ke, s_scan, te);
    const long long pr = block_excl_scan(kr, s_scan, tr);
    long long e = s_carry[0] - total_e + pe, r = s_carry[1] - total_r + pr;   // the carries continue from pass 1
    for (int j = 0; j < V; ++j) {
      const int64_t i = i0 + j;
      if (i >= end) break;
      if (rst(i)) ++r;
      if (keep(i)) {
        if (r < nseen) out[(int64_t)seg[r].start_sub * (S / 8) + (e - seg[r].first_emit)] = d[i];
        ++e;
      }
    }
    __syncthreads();
    if (threadIdx.x == 0) { s_carry[0] += te; s_carry[1] += tr; }
  }
}

// ---- 2. self-synchronising decode: start states and block indices ----
__device__ __forceinline__ int seg_of(const Seg* seg, int nseg, uint32_t j) {   // last g with start_sub <= j
  int lo = 0, hi = nseg - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (seg[mid].start_sub <= j) lo = mid; else hi = mid - 1;
  }
  return lo;
}

struct SubCtx {
  bool active, first;
  int g;
  uint32_t begin, end, seg_end;
};

__device__ __forceinline__ SubCtx sub_ctx(const Img& im, const Seg* seg, int S, int64_t j) {
  SubCtx c;
  c.active = false;
  c.first = false;
  c.g = 0;
  c.begin = c.end = c.seg_end = 0;
  if (j >= im.nsub) return c;
  c.g = seg_of(seg, im.nseg, (uint32_t)j);
  const Seg sg = seg[c.g];
  if (sg.start_sub == 0xffffffffu || (uint32_t)j < sg.start_sub) return c;
  c.seg_end = sg.start_sub * (uint32_t)S + sg.len_bits;
  c.begin = (uint32_t)j * (uint32_t)S;
  c.end = min(c.begin + (uint32_t)S, c.seg_end);
  c.active = c.begin < c.seg_end;
  c.first = (uint32_t)j == sg.start_sub;
  return c;
}

__global__ void __launch_bounds__(kChunk, 4) jpeg_huff_sync(const uint8_t* __restrict__ blob, uint8_t* ws) {
  const Batch& B = *reinterpret_cast<const Batch*>(blob);
  __shared__ int s_ticket;
  __shared__ State s_ex[kChunk];
  __shared__ uint32_t s_cnt[kChunk];
  __shared__ uint8_t s_head[kChunk];
  if (threadIdx.x == 0) s_ticket = atomicAdd(reinterpret_cast<int*>(ws), 1);
  __syncthreads();
  const int t = s_ticket;
  const int i = find_image(chunk_bases(blob, B.n), B.n, t);
  const Img& im = imgs_of(blob)[i];
  const int c = t - chunk_bases(blob, B.n)[i];
  const Seg* seg = reinterpret_cast<const Seg*>(ws + B.ws_seg) + im.seg_base;
  Rec* rec = reinterpret_cast<Rec*>(ws + B.ws_rec);
  const uint32_t* words = reinterpret_cast<const uint32_t*>(ws + B.ws_stream + im.stream_off);
  const int64_t j = (int64_t)c * kChunk + threadIdx.x;
  const SubCtx x = sub_ctx(im, seg, B.sub_bits, j);
  const int tid = threadIdx.x;

  State st = {x.begin, 0};
  State ex = st;
  uint32_t cnt = 0;
  int dummy = 0;
  auto run = [&]() {
    ex = st;
    cnt = x.active ? walk<false>(blob, im, words, ex, x.end, 0, 0, 0, nullptr, dummy) : 0;
  };
  run();
  // Jacobi sweeps: adopt the left neighbour's exit state until no start changes.  Correct whatever the guesses:
  // at the fixed point every start is its left neighbour's exit, and segment-first starts are exact.
  auto settle = [&]() {
    for (;;) {
      s_ex[tid] = ex;
      __syncthreads();
      bool changed = false;
      if (tid > 0 && x.active && !x.first) {
        const State p = s_ex[tid - 1];
        if (p.pos != st.pos || p.bk != st.bk) { st = p; changed = true; }
      }
      if (changed) run();
      if (!__syncthreads_or(changed)) break;
    }
  };
  settle();
  // look-back: the first thread continues from the exit of the CTA before it (ticket order: it is already running)
  uint32_t carry = 0;
  __shared__ int s_need;
  if (tid == 0) s_need = c > 0 && x.active && !x.first;
  __syncthreads();
  if (s_need) {
    __shared__ Rec s_prev;
    if (tid == 0) {
      volatile Rec* pr = rec + (t - 1);
      while (pr->flag == 0) __nanosleep(64);
      __threadfence();
      s_prev.pos = pr->pos;
      s_prev.bk = pr->bk;
      s_prev.count = pr->count;
    }
    __syncthreads();
    carry = s_prev.count;
    bool changed = false;
    if (tid == 0 && (s_prev.pos != st.pos || s_prev.bk != st.bk)) {
      st.pos = s_prev.pos;
      st.bk = s_prev.bk;
      run();
      changed = true;
    }
    if (__syncthreads_or(changed)) settle();
  }
  // segmented exclusive scan of block counts (a segment-first subsequence restarts at 0)
  s_cnt[tid] = cnt;
  s_head[tid] = x.first;
  __syncthreads();
  uint32_t incl = cnt;
  bool head = x.first;
  for (int o = 1; o < kChunk; o <<= 1) {
    uint32_t add = 0;
    bool h = false;
    if (tid >= o) { add = s_cnt[tid - o]; h = s_head[tid - o]; }
    __syncthreads();
    if (tid >= o && !head) { incl += add; head = h; }
    s_cnt[tid] = incl;
    s_head[tid] = head;
    __syncthreads();
  }
  if (!head) incl += carry;
  Sub* sub = reinterpret_cast<Sub*>(ws + B.ws_sub) + im.sub_base;
  if (j < im.nsub) sub[j] = Sub{st.pos, st.bk, incl - cnt, 0};
  if (tid == kChunk - 1) {
    Rec* r = rec + t;
    r->pos = ex.pos;
    r->bk = ex.bk;
    r->count = incl;
    __threadfence();
    atomicExch(&r->flag, 1u);
  }
}

// ---- 3. decode from the synchronised starts, scatter coefficients ----
__global__ void __launch_bounds__(kChunk, 4) jpeg_huff_decode(const uint8_t* __restrict__ blob, uint8_t* ws, int32_t* status) {
  const Batch& B = *reinterpret_cast<const Batch*>(blob);
  const int t = blockIdx.x;
  const int i = find_image(chunk_bases(blob, B.n), B.n, t);
  const Img& im = imgs_of(blob)[i];
  const int c = t - chunk_bases(blob, B.n)[i];
  const Seg* seg = reinterpret_cast<const Seg*>(ws + B.ws_seg) + im.seg_base;
  const int64_t j = (int64_t)c * kChunk + threadIdx.x;
  const SubCtx x = sub_ctx(im, seg, B.sub_bits, j);
  if (!x.active) return;
  const Sub sb = reinterpret_cast<const Sub*>(ws + B.ws_sub)[im.sub_base + j];
  const uint32_t* words = reinterpret_cast<const uint32_t*>(ws + B.ws_stream + im.stream_off);
  const int ri = im.ri ? im.ri : im.total_mcus;
  const uint32_t expected = (uint32_t)(min(ri, im.total_mcus - x.g * ri) * im.bpm);
  int16_t* coef = reinterpret_cast<int16_t*>(ws + B.ws_coef) + (im.coef_off + (int64_t)x.g * ri * im.bpm) * 64;
  State s = {sb.pos, sb.bk};
  int err = 0;
  const int done = walk<true>(blob, im, words, s, x.end, sb.base, expected, x.seg_end, coef, err);
  // the subsequence holding the segment's end must have completed its last block, unless a bad code or index
  // (reported where it occurred) stopped the segment's decode before
  if (x.end == x.seg_end && sb.base + done < expected && sb.pos != kErrPos && s.pos != kErrPos)
    err |= YB_JPEG_TRUNCATED;
  if (err) atomicOr(&status[i], err);
}

// ---- 4. DC prediction: a segmented inclusive scan per component ----
__global__ void __launch_bounds__(kDcThreads) jpeg_dc(const uint8_t* __restrict__ blob, uint8_t* ws) {
  const Batch& B = *reinterpret_cast<const Batch*>(blob);
  const Img& im = imgs_of(blob)[blockIdx.x];
  const int comp = blockIdx.y;
  if (comp >= im.ncomp) return;
  __shared__ int s_v[kDcThreads];
  __shared__ uint8_t s_h[kDcThreads];
  __shared__ int s_carry;
  int off = 0;
  for (int b = 0; b < im.bpm; ++b)
    if (im.blk_comp[b] == comp) { off = b; break; }
  const int per = im.ncomp == 1 ? 1 : im.ch[comp] * im.cv[comp];
  const int64_t cnt = (int64_t)im.total_mcus * per;
  const int ri = im.ri ? im.ri : im.total_mcus;
  int16_t* coef = reinterpret_cast<int16_t*>(ws + B.ws_coef) + im.coef_off * 64;
  if (threadIdx.x == 0) s_carry = 0;
  for (int64_t e0 = 0; e0 < cnt; e0 += blockDim.x) {
    const int64_t e = e0 + threadIdx.x;
    const int64_t m = e / per, b = e % per;
    int v = 0;
    bool h = false;
    int16_t* p = nullptr;
    if (e < cnt) {
      p = coef + (m * im.bpm + off + b) * 64;
      v = *p;
      h = b == 0 && m % ri == 0;
    }
    __syncthreads();
    s_v[threadIdx.x] = v;
    s_h[threadIdx.x] = h;
    __syncthreads();
    bool head = h;
    for (int o = 1; o < (int)blockDim.x; o <<= 1) {
      int add = 0;
      bool hh = false;
      if ((int)threadIdx.x >= o) { add = s_v[threadIdx.x - o]; hh = s_h[threadIdx.x - o]; }
      __syncthreads();
      if ((int)threadIdx.x >= o && !head) { v += add; head = hh; }
      s_v[threadIdx.x] = v;
      s_h[threadIdx.x] = head;
      __syncthreads();
    }
    if (!head) v += s_carry;
    if (p) *p = (int16_t)v;
    __syncthreads();
    if (threadIdx.x == blockDim.x - 1) s_carry = v;
  }
}

// ---- 5. dequantise + ISLOW IDCT, 8 threads per block ----
constexpr int kIdctBlocks = 16;
__device__ __forceinline__ void idct8(const int (&in)[8], int (&o)[8], int shift) {
  int z2 = in[2], z3 = in[6];
  int z1 = (z2 + z3) * 4433;
  const int tmp2 = z1 + z3 * -15137, tmp3 = z1 + z2 * 6270;
  int tmp0 = (in[0] + in[4]) * 8192, tmp1 = (in[0] - in[4]) * 8192;
  const int t10 = tmp0 + tmp3, t13 = tmp0 - tmp3, t11 = tmp1 + tmp2, t12 = tmp1 - tmp2;
  int a0 = in[7], a1 = in[5], a2 = in[3], a3 = in[1];
  z1 = a0 + a3;
  z2 = a1 + a2;
  z3 = a0 + a2;
  int z4 = a1 + a3;
  const int z5 = (z3 + z4) * 9633;
  a0 *= 2446;
  a1 *= 16819;
  a2 *= 25172;
  a3 *= 12299;
  z1 *= -7373;
  z2 *= -20995;
  z3 = z3 * -16069 + z5;
  z4 = z4 * -3196 + z5;
  a0 += z1 + z3;
  a1 += z2 + z4;
  a2 += z2 + z3;
  a3 += z1 + z4;
  const int r = 1 << (shift - 1);
  o[0] = (t10 + a3 + r) >> shift;
  o[7] = (t10 - a3 + r) >> shift;
  o[1] = (t11 + a2 + r) >> shift;
  o[6] = (t11 - a2 + r) >> shift;
  o[2] = (t12 + a1 + r) >> shift;
  o[5] = (t12 - a1 + r) >> shift;
  o[3] = (t13 + a0 + r) >> shift;
  o[4] = (t13 - a0 + r) >> shift;
}

__global__ void __launch_bounds__(kIdctBlocks * 8) jpeg_idct(const uint8_t* __restrict__ blob, uint8_t* ws) {
  const Batch& B = *reinterpret_cast<const Batch*>(blob);
  const Img& im = imgs_of(blob)[blockIdx.y];
  __shared__ int s_ws[kIdctBlocks][8][9];
  const int lb = threadIdx.x >> 3, r = threadIdx.x & 7;
  const int64_t idx = (int64_t)blockIdx.x * kIdctBlocks + lb;
  const int64_t nblk = (int64_t)im.total_mcus * im.bpm;
  if (idx >= nblk) return;   // whole 8-thread groups leave together
  const int64_t m = idx / im.bpm;
  const int b = (int)(idx % im.bpm);
  const int comp = im.blk_comp[b];
  int64_t bx, by;
  if (im.ncomp == 1) { bx = m % im.mcus_x; by = m / im.mcus_x; }
  else { bx = (m % im.mcus_x) * im.ch[comp] + im.blk_x[b]; by = (m / im.mcus_x) * im.cv[comp] + im.blk_y[b]; }
  const int16_t* cf = reinterpret_cast<const int16_t*>(ws + B.ws_coef) + (im.coef_off + idx) * 64;
  int in[8], o[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) in[k] = (int)cf[k * 8 + r] * (int)im.q[comp][k * 8 + r];   // column r
  idct8(in, o, 11);
#pragma unroll
  for (int k = 0; k < 8; ++k) s_ws[lb][k][r] = o[k];
  __syncwarp(0xffu << (threadIdx.x & 24));
#pragma unroll
  for (int k = 0; k < 8; ++k) in[k] = s_ws[lb][r][k];                                     // row r
  idct8(in, o, 18);
  uint32_t w0 = 0, w1 = 0;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    w0 |= (uint32_t)(min(max(o[k], -128), 127) + 128) << (8 * k);
    w1 |= (uint32_t)(min(max(o[k + 4], -128), 127) + 128) << (8 * k);
  }
  const int64_t pitch = (int64_t)im.pw[comp] * 8;
  uint8_t* dst = ws + B.ws_planes + im.plane_off[comp] + (by * 8 + r) * pitch + bx * 8;
  *reinterpret_cast<uint2*>(dst) = make_uint2(w0, w1);
}

// ---- 6. upsample + colour + orientation ----
__device__ __forceinline__ int sample(const uint8_t* p, int64_t pitch, int y, int x) { return p[(int64_t)y * pitch + x]; }

// component `c` at full-resolution pixel (y, x): libjpeg-turbo's fancy upsampling (jdsample.c), box when the
// downsampled width is 2 or less for the horizontal cases
__device__ __forceinline__ int upsampled(const Img& im, const uint8_t* planes, int c, int y, int x) {
  const uint8_t* p = planes + im.plane_off[c];
  const int64_t pitch = (int64_t)im.pw[c] * 8;
  const int hr = im.hmax / im.ch[c], vr = im.vmax / im.cv[c];
  const int dw = im.dw[c], dh = im.dh[c];
  if (im.ncomp == 1 || (hr == 1 && vr == 1)) return sample(p, pitch, y, x);
  if (hr == 1) {   // h1v2
    const int i = y >> 1, odd = y & 1;
    const int nb = odd ? min(i + 1, dh - 1) : max(i - 1, 0);
    return (3 * sample(p, pitch, i, x) + sample(p, pitch, nb, x) + 1 + odd) >> 2;
  }
  const int i = x >> 1, odd = x & 1;
  if (dw <= 2) return sample(p, pitch, vr == 2 ? y >> 1 : y, i);
  const int j = odd ? min(i + 1, dw - 1) : max(i - 1, 0);
  if (vr == 1)   // h2v1
    return (3 * sample(p, pitch, y, i) + sample(p, pitch, y, j) + 1 + odd) >> 2;
  const int r = y >> 1;   // h2v2
  const int nb = (y & 1) ? min(r + 1, dh - 1) : max(r - 1, 0);
  const int cs_i = 3 * sample(p, pitch, r, i) + sample(p, pitch, nb, i);
  const int cs_j = 3 * sample(p, pitch, r, j) + sample(p, pitch, nb, j);
  return (3 * cs_i + cs_j + 8 - odd) >> 4;
}

__global__ void __launch_bounds__(256) jpeg_color(const uint8_t* __restrict__ blob, const uint8_t* ws,
                                                  uint8_t* out_pixels, int64_t* out_desc) {
  const Batch& B = *reinterpret_cast<const Batch*>(blob);
  const Img& im = imgs_of(blob)[blockIdx.y];
  if (blockIdx.x == 0 && threadIdx.x < 4) {
    const int q = threadIdx.x;
    out_desc[blockIdx.y * 4 + q] = q == 0 ? im.pix_off : q == 1 ? im.out_h : q == 2 ? im.out_w : 3 * (int64_t)im.out_w;
  }
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (int64_t)im.H * im.W) return;
  const int y = (int)(e / im.W), x = (int)(e % im.W);
  const uint8_t* planes = ws + B.ws_planes;
  int bb, gg, rr;
  const int Y = upsampled(im, planes, 0, y, x);
  if (im.ncomp == 1) {
    bb = gg = rr = Y;
  } else {
    const int cb = upsampled(im, planes, 1, y, x) - 128, cr = upsampled(im, planes, 2, y, x) - 128;
    rr = Y + ((91881 * cr + 32768) >> 16);
    gg = Y + ((-22554 * cb + 32768 - 46802 * cr) >> 16);
    bb = Y + ((116130 * cb + 32768) >> 16);
    rr = min(max(rr, 0), 255);
    gg = min(max(gg, 0), 255);
    bb = min(max(bb, 0), 255);
  }
  const int H = im.H, W = im.W;
  int oy = y, ox = x;
  switch (im.orient) {
    case 2: ox = W - 1 - x; break;
    case 3: oy = H - 1 - y; ox = W - 1 - x; break;
    case 4: oy = H - 1 - y; break;
    case 5: oy = x; ox = y; break;
    case 6: oy = x; ox = H - 1 - y; break;
    case 7: oy = W - 1 - x; ox = H - 1 - y; break;
    case 8: oy = W - 1 - x; ox = y; break;
    default: break;
  }
  uint8_t* d = out_pixels + im.pix_off + ((int64_t)oy * im.out_w + ox) * 3;
  d[0] = (uint8_t)bb;
  d[1] = (uint8_t)gg;
  d[2] = (uint8_t)rr;
}

}  // namespace

// ---------------------------------------------------------------------------------------------------------------
// host: pack
// ---------------------------------------------------------------------------------------------------------------
namespace {

struct Plan {   // pack's layout of one batch
  std::vector<Layout> L;
  std::vector<Img> img;
  std::vector<int32_t> chunk_base;
  Batch B;
  int64_t blob_bytes;
  std::vector<int64_t> tab_pos;   // blob offset of each image's tables
};

static int plan_batch(const void* const* data, const size_t* bytes, int n, Plan& P) {
  YB_REQUIRE(data && bytes && n >= 1 && n <= 65535, "yb_jpeg_pack: need 1..65535 images and their sizes");
  const int S = sub_bits_option();
  YB_REQUIRE(S >= 32 && S <= 65536 && S % 32 == 0, "YB_JPEG_SUBSEQ_BITS must be a multiple of 32 in 32..65536, got %d", S);
  P.L.resize(n);
  P.img.assign(n, Img{});
  P.chunk_base.resize(n);
  P.tab_pos.resize(n);
  memset(&P.B, 0, sizeof(P.B));
  int64_t off = align16(sizeof(Batch) + sizeof(Img) * (int64_t)n + 4 * (int64_t)n);
  int64_t stream = 0, nsub = 0, nseg = 0, blocks = 0, planes = 0, pix = 0, chunks = 0, max_blocks = 0, max_pix = 0;
  for (int i = 0; i < n; ++i) {
    Layout& L = P.L[i];
    const int rc = layout(static_cast<const uint8_t*>(data[i]), bytes[i], L);
    if (rc) {
      char why[400];
      snprintf(why, sizeof(why), "%s", yb_last_error_string());
      set_error("image %d: %s", i, why);
      return rc;
    }
    const Parsed& Q = L.P;
    Img& m = P.img[i];
    const int64_t dlen = (int64_t)bytes[i] - (int64_t)Q.scan_start;
    if (dlen >= (int64_t(1) << 28)) { set_error("image %d: more than 256 MB of entropy-coded data", i); return YB_ERR_UNSUPPORTED; }
    m.data_len = dlen;
    m.ncomp = Q.nf;
    m.H = Q.H;
    m.W = Q.W;
    m.orient = Q.orient;
    m.out_h = Q.orient >= 5 ? Q.W : Q.H;
    m.out_w = Q.orient >= 5 ? Q.H : Q.W;
    m.hmax = L.hmax;
    m.vmax = L.vmax;
    m.mcus_x = L.mcus_x;
    m.total_mcus = L.mcus_x * L.mcus_y;
    m.ri = Q.ri;
    m.nseg = Q.ri ? (m.total_mcus + Q.ri - 1) / Q.ri : 1;
    m.bpm = L.bpm;
    int b = 0;
    for (int c = 0; c < Q.nf; ++c) {
      const int hh = Q.nf == 1 ? 1 : Q.h[c], vv = Q.nf == 1 ? 1 : Q.v[c];
      m.ch[c] = hh;
      m.cv[c] = vv;
      m.pw[c] = L.pw[c];
      m.dw[c] = L.dw[c];
      m.dh[c] = L.dh[c];
      for (int yy = 0; yy < vv; ++yy)
        for (int xx = 0; xx < hh; ++xx) { m.blk_comp[b] = (int8_t)c; m.blk_x[b] = (int8_t)xx; m.blk_y[b] = (int8_t)yy; ++b; }
      for (int k = 0; k < 64; ++k) m.q[c][k] = Q.q[Q.tq[c]][k];
      m.plane_off[c] = planes;
      planes += align16((int64_t)L.pw[c] * 8 * L.ph[c] * 8);
    }
    const int64_t img_subs = (dlen * 8 + S - 1) / S + m.nseg;
    if (img_subs * S >= (int64_t(1) << 32)) {   // bit positions in the destuffed stream are 32-bit
      set_error("image %d: %lld restart segments of %lld entropy-coded bytes need more than 2^32 stream bits at "
                "YB_JPEG_SUBSEQ_BITS %d", i, (long long)m.nseg, (long long)dlen, S);
      return YB_ERR_UNSUPPORTED;
    }
    m.nsub = (int32_t)img_subs;
    m.stream_off = stream;
    stream += align16((int64_t)m.nsub * (S / 8) + 16);
    m.sub_base = nsub;
    nsub += m.nsub;
    m.seg_base = nseg;
    nseg += m.nseg;
    m.coef_off = blocks;
    const int64_t nb = (int64_t)m.total_mcus * m.bpm;
    blocks += nb;
    max_blocks = nb > max_blocks ? nb : max_blocks;
    max_pix = (int64_t)m.H * m.W > max_pix ? (int64_t)m.H * m.W : max_pix;
    m.pix_off = pix;
    pix += align16((int64_t)m.out_h * m.out_w * 3);
    m.chunk_base = (int32_t)chunks;
    P.chunk_base[i] = (int32_t)chunks;
    chunks += (m.nsub + kChunk - 1) / kChunk;
    YB_REQUIRE(chunks < (int64_t(1) << 31), "yb_jpeg_pack: batch too large");
    // tables: one HuffTab per distinct (class, id) the scan uses, then the entropy bytes
    P.tab_pos[i] = off;
    int used[2][4] = {{-1, -1, -1, -1}, {-1, -1, -1, -1}};
    int ntab = 0;
    for (int c = 0; c < Q.nf; ++c)
      for (int k = 0; k < 2; ++k) {
        const int id = k ? Q.ta[c] : Q.td[c];
        if (used[k][id] < 0) used[k][id] = ntab++;
        m.tab_off[c][k] = off + (int64_t)sizeof(HuffTab) * used[k][id];
      }
    L.ntab = ntab;
    off += (int64_t)sizeof(HuffTab) * ntab;
    m.data_off = off;
    off = align16(off + dlen);
  }
  Batch& B = P.B;
  B.magic = kMagic;
  B.n = n;
  B.sub_bits = S;
  B.nchunks = (int32_t)chunks;
  B.ws_rec = 256;
  B.ws_seg = align16(B.ws_rec + 16 * chunks);
  B.ws_sub = align16(B.ws_seg + 16 * nseg);
  B.ws_stream = align16(B.ws_sub + 16 * nsub);
  B.ws_coef = align16(B.ws_stream + stream);
  B.ws_planes = align16(B.ws_coef + 128 * blocks);
  B.ws_bytes = align16(B.ws_planes + planes + 16);
  B.max_blocks = max_blocks;
  B.max_pixels = max_pix;
  B.pixel_bytes = pix;
  P.blob_bytes = off;
  return YB_OK;
}

static int check_blob(const void* host_blob, int n, const Batch*& B) {
  YB_REQUIRE(host_blob, "jpeg: null host blob");
  B = static_cast<const Batch*>(host_blob);
  YB_REQUIRE(B->magic == kMagic, "jpeg: host blob was not written by yb_jpeg_pack");
  YB_REQUIRE(B->n == n, "jpeg: the blob holds %d images, not %d", B->n, n);
  return YB_OK;
}

}  // namespace
}  // namespace yb

using namespace yb;

extern "C" int yb_jpeg_parse(const void* data, size_t bytes, yb_jpeg_info* info) {
  YB_REQUIRE(data && info, "yb_jpeg_parse: null argument");
  Layout L;
  const int rc = layout(static_cast<const uint8_t*>(data), bytes, L);
  if (rc) return rc;
  const Parsed& P = L.P;
  info->height = P.orient >= 5 ? P.W : P.H;
  info->width = P.orient >= 5 ? P.H : P.W;
  info->src_height = P.H;
  info->src_width = P.W;
  info->components = P.nf;
  info->h_samp = P.nf == 3 ? P.h[0] : 1;
  info->v_samp = P.nf == 3 ? P.v[0] : 1;
  info->restart_interval = P.ri;
  info->orientation = P.orient;
  info->mode = P.mode;
  return YB_OK;
}

extern "C" int yb_jpeg_pack_bytes(const void* const* data, const size_t* bytes, int n, size_t* blob_bytes) {
  YB_REQUIRE(blob_bytes, "yb_jpeg_pack_bytes: null blob_bytes");
  Plan P;
  const int rc = plan_batch(data, bytes, n, P);
  if (rc) return rc;
  *blob_bytes = (size_t)P.blob_bytes;
  return YB_OK;
}

extern "C" int yb_jpeg_pack(const void* const* data, const size_t* bytes, int n, void* host_blob, size_t blob_bytes,
                            int64_t* desc_host) {
  YB_REQUIRE(host_blob, "yb_jpeg_pack: null host_blob");
  Plan P;
  int rc = plan_batch(data, bytes, n, P);
  if (rc) return rc;
  YB_REQUIRE((int64_t)blob_bytes >= P.blob_bytes, "yb_jpeg_pack: blob of %zu bytes, %lld needed", blob_bytes,
             (long long)P.blob_bytes);
  uint8_t* o = static_cast<uint8_t*>(host_blob);
  memcpy(o, &P.B, sizeof(Batch));
  memcpy(o + sizeof(Batch), P.img.data(), sizeof(Img) * (size_t)n);
  memcpy(o + sizeof(Batch) + sizeof(Img) * (size_t)n, P.chunk_base.data(), 4 * (size_t)n);
  for (int i = 0; i < n; ++i) {
    const Parsed& Q = P.L[i].P;
    const Img& m = P.img[i];
    for (int c = 0; c < Q.nf; ++c)
      for (int k = 0; k < 2; ++k) {
        const int id = k ? Q.ta[c] : Q.td[c];
        HuffTab t;
        build_table(Q.bits[k][id], Q.vals[k][id], t);   // validated by layout()
        memcpy(o + m.tab_off[c][k], &t, sizeof(t));
      }
    memcpy(o + m.data_off, static_cast<const uint8_t*>(data[i]) + Q.scan_start, (size_t)m.data_len);
    if (desc_host) {
      desc_host[4 * i] = m.pix_off;
      desc_host[4 * i + 1] = m.out_h;
      desc_host[4 * i + 2] = m.out_w;
      desc_host[4 * i + 3] = 3 * (int64_t)m.out_w;
    }
  }
  return YB_OK;
}

extern "C" int yb_jpeg_workspace_bytes(const void* host_blob, int n, size_t* bytes, size_t* pixel_bytes) {
  const Batch* B;
  const int rc = check_blob(host_blob, n, B);
  if (rc) return rc;
  YB_REQUIRE(bytes, "yb_jpeg_workspace_bytes: null bytes");
  *bytes = (size_t)B->ws_bytes;
  if (pixel_bytes) *pixel_bytes = (size_t)B->pixel_bytes;
  return YB_OK;
}

extern "C" int yb_jpeg_decode(const void* dev_blob, const void* host_blob, int n, uint8_t* out_pixels, int64_t* out_desc,
                              int32_t* status, void* workspace, size_t workspace_bytes, void* stream) {
  const Batch* B;
  int rc = check_blob(host_blob, n, B);
  if (rc) return rc;
  YB_REQUIRE(dev_blob && out_pixels && out_desc && status, "yb_jpeg_decode: null device pointer");
  YB_REQUIRE(workspace, "yb_jpeg_decode: null workspace");
  if (workspace_bytes < (size_t)B->ws_bytes) {
    set_error("yb_jpeg_decode: workspace of %zu bytes, %lld needed", workspace_bytes, (long long)B->ws_bytes);
    return YB_ERR_WORKSPACE;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const uint8_t* blob = static_cast<const uint8_t*>(dev_blob);
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  YB_CUDA(cudaMemsetAsync(status, 0, sizeof(int32_t) * (size_t)n, st));
  YB_CUDA(cudaMemsetAsync(ws, 0, (size_t)B->ws_planes, st));
  jpeg_destuff<<<n, kDestuffThreads, 0, st>>>(blob, ws, status);
  YB_CUDA(cudaGetLastError());
  jpeg_huff_sync<<<B->nchunks, kChunk, 0, st>>>(blob, ws);
  YB_CUDA(cudaGetLastError());
  jpeg_huff_decode<<<B->nchunks, kChunk, 0, st>>>(blob, ws, status);
  YB_CUDA(cudaGetLastError());
  jpeg_dc<<<dim3(n, 3), kDcThreads, 0, st>>>(blob, ws);
  YB_CUDA(cudaGetLastError());
  jpeg_idct<<<dim3((unsigned)((B->max_blocks + kIdctBlocks - 1) / kIdctBlocks), n), kIdctBlocks * 8, 0, st>>>(blob, ws);
  YB_CUDA(cudaGetLastError());
  jpeg_color<<<dim3((unsigned)((B->max_pixels + 255) / 256), n), 256, 0, st>>>(blob, ws, out_pixels, out_desc);
  YB_CUDA(cudaGetLastError());
  return YB_OK;
}
