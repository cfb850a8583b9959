// Batched baseline JPEG encode (replaces cv2.imwrite / cv2.imencode('.jpg'), test_single_image.py:85): files equal
// byte for byte to cv2.imencode of OpenCV 4.13 / libjpeg-turbo 3.1 (DESIGN.md §2 states the rules).
//
// Host: resolve the OpenCV parameters, build the header bytes, quantisation reciprocals and MCU geometry of every
// image and pack them with the Huffman code tables into one blob (the batch's one H2D copy).  Device, one launch per
// stage for the whole batch:
//   1. enc_fdct      one thread per block: colour conversion, edge replication, downsampling, ISLOW FDCT and
//                    reciprocal quantisation -> int16 coefficients in zigzag order; dummy blocks get AC zero and
//                    the DC of the block before them in their MCU.
//   2. enc_count     one thread per block: DC difference and Huffman bit count; per-segment bit totals.
//   3. enc_scan      one CTA per image: segment starts (each on a 1024-bit chunk boundary), a segmented scan of
//                    the block bit counts, and zeroing of the image's word stream.
//   4. enc_emit      one thread per block: codes into the 32-bit word stream (MSB first, atomicOr on the words a
//                    block shares), segment ends padded with 1-bits.
//   5. enc_ffcount   one warp per 128-byte chunk: its 0xFF bytes, added to its segment's total.
//   6. enc_layout    one CTA per image: segmented scan of chunk 0xFF counts; scan of the stuffed segment lengths.
//   7. enc_files     one CTA: file offsets and lengths.
//   8. enc_assemble  header, stuffed segments, RSTn markers and EOI of every file.
#include <string.h>

#include <algorithm>
#include <vector>

#include "common.cuh"

namespace yb {
namespace {

constexpr uint32_t kEncMagic = 0x4a454e31;   // "JEN1"
constexpr int kBlockThreads = 128;
constexpr int kScanThreads = 1024;
constexpr int kChunkBits = 1024;             // segments start on a chunk: a warp's 32 words never span two
constexpr int kMaxBlockBits = 27 + 63 * 26;  // longest DC code + size bits, 63 x (longest AC code + size bits)
constexpr int kMaxHeader = 640;

constexpr uint8_t kZigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,
                                 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28,
                                 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
                                 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// ITU T.81 Annex K: K.1 base quantisation tables (natural order), K.3 standard Huffman tables
const uint8_t kBaseQ[2][64] = {
    {16, 11, 10, 16, 24,  40,  51,  61,  12, 12, 14, 19, 26,  58,  60,  55,  14, 13, 16, 24, 40,  57,
     69, 56, 14, 17, 22,  29,  51,  87,  80, 62, 18, 22, 37,  56,  68,  109, 103, 77, 24, 35, 55, 64,
     81, 104, 113, 92, 49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99},
    {17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99,
     99, 99, 47, 66, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99,
     99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99}};
const uint8_t kDcBits[2][16] = {{0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0}, {0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0}};
const uint8_t kAcBits[2][16] = {{0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 125}, {0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 119}};
const uint8_t kAcVals[2][162] = {
    {0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14,
     0x32, 0x81, 0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09,
     0x0a, 0x16, 0x17, 0x18, 0x19, 0x1a, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a,
     0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65,
     0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88,
     0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9,
     0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca,
     0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea,
     0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa},
    {0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22, 0x32,
     0x81, 0x08, 0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16,
     0x24, 0x34, 0xe1, 0x25, 0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x35, 0x36, 0x37, 0x38, 0x39,
     0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64,
     0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x82, 0x83, 0x84, 0x85, 0x86,
     0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7,
     0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8,
     0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9,
     0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa}};

struct EncImg {
  uint64_t src;                 // device address of row 0
  int64_t pitch;
  int32_t H, W, channels, ncomp;
  int32_t hmax, vmax, mcus_x, mcus_y;
  int32_t bpm, ri, nseg, hdr_len;   // blocks per MCU, restart interval in MCUs (0: one segment)
  int64_t nblocks, blk_base, seg_base, word_base, chunk_base, max_chunks, hdr_off;
  int32_t ch[3], cv[3], wib[3], hib[3];
  int8_t blk_comp[6], blk_x[6], blk_y[6], pad[6];
  uint16_t recip[2][64], corr[2][64];   // natural order, per quantisation table
  uint8_t shift[2][64];
};

struct EncBatch {
  uint32_t magic;
  int32_t n;
  int64_t total_blocks, total_segs, total_chunks, max_blocks, max_chunks, out_bytes;
  int64_t ws_coef, ws_bits, ws_off, ws_seg_bits, ws_seg_ff, ws_seg_start, ws_seg_out, ws_img, ws_words, ws_chunk_ff,
      ws_chunk_seg, ws_chunk_before, ws_bytes;
  uint32_t dc_code[2][16];     // (code << 8) | length by symbol
  uint32_t ac_code[2][256];
};

struct Resolved { int s0, s1, h, v, ri, nt; };

static int quality_scale(int q) {   // libjpeg's jpeg_quality_scaling
  q = q < 1 ? 1 : q > 100 ? 100 : q;
  return q < 50 ? 5000 / q : 200 - 2 * q;
}

static int resolve(const yb_jpeg_enc_image& im, Resolved& R) {
  YB_REQUIRE(im.height >= 1 && im.height <= 65535 && im.width >= 1 && im.width <= 65535,
             "size %d x %d is outside 1..65535", im.height, im.width);
  YB_REQUIRE(im.channels == 1 || im.channels == 3, "%d channels: need 1 (grey) or 3 (BGR)", im.channels);
  YB_REQUIRE(im.pitch >= (int64_t)im.width * im.channels, "row pitch %lld is less than width x channels",
             (long long)im.pitch);
  int h, v;
  switch (im.sampling) {
    case YB_JPEG_SAMPLING_411: h = 4, v = 1; break;
    case YB_JPEG_SAMPLING_420: h = 2, v = 2; break;
    case YB_JPEG_SAMPLING_422: h = 2, v = 1; break;
    case YB_JPEG_SAMPLING_440: h = 1, v = 2; break;
    case YB_JPEG_SAMPLING_444: h = 1, v = 1; break;
    default: YB_REQUIRE(false, "sampling 0x%x is not one of the IMWRITE_JPEG_SAMPLING_FACTOR values", im.sampling);
  }
  // OpenCV clamps quality to 0..100 (libjpeg then to 1..100).  A luma quality >= 0 replaces quality and, when no
  // chroma quality is given, the chroma quality; a chroma quality alone is ignored.  Unequal ones disable
  // subsampling.
  int q = im.quality < 0 ? 0 : im.quality > 100 ? 100 : im.quality;
  R.s0 = R.s1 = quality_scale(q);
  if (im.luma_quality >= 0) {
    const int lq = im.luma_quality > 100 ? 100 : im.luma_quality;
    const int cq = im.chroma_quality >= 0 ? (im.chroma_quality > 100 ? 100 : im.chroma_quality) : lq;
    R.s0 = quality_scale(lq);
    R.s1 = quality_scale(cq);
    if (lq != cq) h = v = 1;
  }
  if (im.channels == 1) h = v = 1;
  R.h = h;
  R.v = v;
  R.ri = im.restart_interval < 0 ? 0 : im.restart_interval > 65535 ? 65535 : im.restart_interval;
  R.nt = im.channels == 1 ? 1 : 2;
  return YB_OK;
}

static void quant_table(int t, int scale, uint8_t out[64]) {
  for (int i = 0; i < 64; ++i) {
    int q = (kBaseQ[t][i] * scale + 50) / 100;
    out[i] = (uint8_t)(q < 1 ? 1 : q > 255 ? 255 : q);
  }
}

// libjpeg-turbo's compute_reciprocal for the divisor 8q: |x| / 8q rounded half up is ((|x| + corr) * recip) >> shift
static void reciprocal(int q, uint16_t& recip, uint16_t& corr, uint8_t& shift) {
  const uint32_t d = 8u * (uint32_t)q;
  int b = 31 - __builtin_clz(d);
  int r = 16 + b;
  uint32_t fq = (uint32_t)((1ull << r) / d), fr = (uint32_t)((1ull << r) % d), c = d / 2;
  if (fr == 0) { fq >>= 1; --r; }
  else if (fr <= d / 2) ++c;
  else ++fq;
  recip = (uint16_t)fq;
  corr = (uint16_t)c;
  shift = (uint8_t)r;
}

static size_t build_header(const yb_jpeg_enc_image& im, const Resolved& R, uint8_t* o) {
  size_t p = 0;
  auto b = [&](int v) { o[p++] = (uint8_t)v; };
  auto seg = [&](int marker, int len) { b(0xFF); b(marker); b((len + 2) >> 8); b((len + 2) & 255); };
  b(0xFF); b(0xD8);
  static const uint8_t jfif[14] = {'J', 'F', 'I', 'F', 0, 1, 1, 0, 0, 1, 0, 1, 0, 0};
  seg(0xE0, 14);
  for (int i = 0; i < 14; ++i) b(jfif[i]);
  for (int t = 0; t < R.nt; ++t) {
    uint8_t q[64];
    quant_table(t, t ? R.s1 : R.s0, q);
    seg(0xDB, 65);
    b(t);
    for (int k = 0; k < 64; ++k) b(q[kZigzag[k]]);
  }
  const int nc = im.channels == 1 ? 1 : 3;
  seg(0xC0, 6 + 3 * nc);
  b(8); b(im.height >> 8); b(im.height & 255); b(im.width >> 8); b(im.width & 255); b(nc);
  for (int c = 0; c < nc; ++c) { b(c + 1); b(c ? 0x11 : (R.h << 4 | R.v)); b(c ? 1 : 0); }
  for (int t = 0; t < R.nt; ++t) {
    seg(0xC4, 17 + 12);
    b(t);
    for (int k = 0; k < 16; ++k) b(kDcBits[t][k]);
    for (int k = 0; k < 12; ++k) b(k);
    seg(0xC4, 17 + 162);
    b(0x10 | t);
    for (int k = 0; k < 16; ++k) b(kAcBits[t][k]);
    for (int k = 0; k < 162; ++k) b(kAcVals[t][k]);
  }
  if (R.ri) { seg(0xDD, 2); b(R.ri >> 8); b(R.ri & 255); }
  seg(0xDA, 4 + 2 * nc);
  b(nc);
  for (int c = 0; c < nc; ++c) { b(c + 1); b(c ? 0x11 : 0x00); }
  b(0); b(63); b(0);
  return p;
}

static void huff_codes(const uint8_t bits[16], const uint8_t* vals, uint32_t* table) {   // Annex C
  uint32_t code = 0;
  int k = 0;
  for (int len = 1; len <= 16; ++len) {
    for (int i = 0; i < bits[len - 1]; ++i, ++k) table[vals[k]] = code++ << 8 | (uint32_t)len;
    code <<= 1;
  }
}

struct EncPlan {
  std::vector<EncImg> img;
  std::vector<uint8_t> hdr;
  EncBatch B;
  int64_t blob_bytes;
};

static inline int64_t align16(int64_t v) { return (v + 15) & ~int64_t(15); }

static int plan_enc(const yb_jpeg_enc_image* images, int n, EncPlan& P) {
  YB_REQUIRE(images && n >= 1 && n <= 65535, "yb_jpeg_enc_pack: need 1..65535 images");
  P.img.assign(n, EncImg{});
  P.hdr.clear();
  memset(&P.B, 0, sizeof(P.B));
  const int64_t hdr0 = align16(sizeof(EncBatch) + sizeof(EncImg) * (int64_t)n);
  int64_t blocks = 0, segs = 0, chunks = 0, max_blocks = 0, max_chunks = 0, out = 0;
  for (int i = 0; i < n; ++i) {
    const yb_jpeg_enc_image& im = images[i];
    Resolved R;
    if (resolve(im, R)) {
      char why[400];
      snprintf(why, sizeof(why), "%s", yb_last_error_string());
      set_error("image %d: %s", i, why);
      return YB_ERR_INVALID_ARGUMENT;
    }
    if (!im.pixels) { set_error("image %d: null pixels", i); return YB_ERR_INVALID_ARGUMENT; }
    EncImg& m = P.img[i];
    m.src = (uint64_t)(uintptr_t)im.pixels;
    m.pitch = im.pitch;
    m.H = im.height;
    m.W = im.width;
    m.channels = im.channels;
    m.ncomp = im.channels == 1 ? 1 : 3;
    m.hmax = R.h;
    m.vmax = R.v;
    m.mcus_x = (im.width + 8 * R.h - 1) / (8 * R.h);
    m.mcus_y = (im.height + 8 * R.v - 1) / (8 * R.v);
    int b = 0;
    for (int c = 0; c < m.ncomp; ++c) {
      const int hh = c ? 1 : R.h, vv = c ? 1 : R.v;
      m.ch[c] = hh;
      m.cv[c] = vv;
      m.wib[c] = (int32_t)(((int64_t)im.width * hh + 8 * R.h - 1) / (8 * R.h));
      m.hib[c] = (int32_t)(((int64_t)im.height * vv + 8 * R.v - 1) / (8 * R.v));
      for (int y = 0; y < vv; ++y)
        for (int x = 0; x < hh; ++x) { m.blk_comp[b] = (int8_t)c; m.blk_x[b] = (int8_t)x; m.blk_y[b] = (int8_t)y; ++b; }
    }
    m.bpm = b;
    m.ri = R.ri;
    const int64_t mcus = (int64_t)m.mcus_x * m.mcus_y;
    m.nseg = (int32_t)(R.ri ? (mcus + R.ri - 1) / R.ri : 1);
    m.nblocks = mcus * m.bpm;
    for (int t = 0; t < R.nt; ++t) {
      uint8_t q[64];
      quant_table(t, t ? R.s1 : R.s0, q);
      for (int k = 0; k < 64; ++k) reciprocal(q[k], m.recip[t][k], m.corr[t][k], m.shift[t][k]);
    }
    uint8_t h[kMaxHeader];
    m.hdr_len = (int32_t)build_header(im, R, h);
    m.hdr_off = hdr0 + (int64_t)P.hdr.size();
    P.hdr.insert(P.hdr.end(), h, h + m.hdr_len);
    // word stream bound: every block at its longest, every segment padded to a chunk
    const int64_t img_chunks = (m.nblocks * kMaxBlockBits + kChunkBits - 1) / kChunkBits + m.nseg;
    m.blk_base = blocks;
    m.seg_base = segs;
    m.chunk_base = chunks;
    m.word_base = chunks * (kChunkBits / 32);
    m.max_chunks = img_chunks;
    blocks += m.nblocks;
    segs += m.nseg;
    chunks += img_chunks;
    max_blocks = m.nblocks > max_blocks ? m.nblocks : max_blocks;
    max_chunks = img_chunks > max_chunks ? img_chunks : max_chunks;
    // file bound: header, every data byte stuffed, an RSTn per segment, EOI
    out += m.hdr_len + 2 * ((m.nblocks * kMaxBlockBits + 7) / 8 + m.nseg) + 2 * m.nseg + 2;
  }
  EncBatch& B = P.B;
  B.magic = kEncMagic;
  B.n = n;
  B.total_blocks = blocks;
  B.total_segs = segs;
  B.total_chunks = chunks;
  B.max_blocks = max_blocks;
  B.max_chunks = max_chunks;
  B.out_bytes = align16(out);
  B.ws_coef = 0;
  B.ws_bits = align16(B.ws_coef + 128 * blocks);
  B.ws_off = align16(B.ws_bits + 4 * blocks);
  B.ws_seg_bits = align16(B.ws_off + 8 * blocks);
  B.ws_seg_ff = B.ws_seg_bits + 8 * segs;               // zeroed together with seg_bits
  B.ws_seg_start = align16(B.ws_seg_ff + 8 * segs);
  B.ws_seg_out = align16(B.ws_seg_start + 8 * segs);
  B.ws_img = align16(B.ws_seg_out + 8 * segs);          // per image: used chunks, file length
  B.ws_words = align16(B.ws_img + 16 * (int64_t)n);
  B.ws_chunk_ff = align16(B.ws_words + 128 * chunks);
  B.ws_chunk_seg = align16(B.ws_chunk_ff + 4 * chunks);
  B.ws_chunk_before = align16(B.ws_chunk_seg + 4 * chunks);
  B.ws_bytes = align16(B.ws_chunk_before + 8 * chunks);
  for (int t = 0; t < 2; ++t) {
    static const uint8_t dc_vals[12] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11};
    huff_codes(kDcBits[t], dc_vals, B.dc_code[t]);
    huff_codes(kAcBits[t], kAcVals[t], B.ac_code[t]);
  }
  P.blob_bytes = align16(hdr0 + (int64_t)P.hdr.size());
  return YB_OK;
}

static int check_enc_blob(const void* host_blob, int n, const EncBatch*& B) {
  YB_REQUIRE(host_blob, "jpeg encode: null host blob");
  B = static_cast<const EncBatch*>(host_blob);
  YB_REQUIRE(B->magic == kEncMagic, "jpeg encode: host blob was not written by yb_jpeg_enc_pack");
  YB_REQUIRE(B->n == n, "jpeg encode: the blob holds %d images, not %d", B->n, n);
  return YB_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// device
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ const EncImg& enc_img(const uint8_t* blob, int i) {
  return reinterpret_cast<const EncImg*>(blob + sizeof(EncBatch))[i];
}

__device__ __forceinline__ int descale(int x, int n) { return (x + (1 << (n - 1))) >> n; }

// jfdctint.c: one 1-D pass over 8 values with stride s; pass 0 keeps PASS1_BITS (2) of extra precision
template <int kPass>
__device__ __forceinline__ void fdct_1d(int* d, int s) {
  const int t0 = d[0] + d[7 * s], t7 = d[0] - d[7 * s], t1 = d[s] + d[6 * s], t6 = d[s] - d[6 * s];
  const int t2 = d[2 * s] + d[5 * s], t5 = d[2 * s] - d[5 * s], t3 = d[3 * s] + d[4 * s], t4 = d[3 * s] - d[4 * s];
  const int t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
  constexpr int sh = kPass == 0 ? 11 : 15;
  if (kPass == 0) { d[0] = (t10 + t11) * 4; d[4 * s] = (t10 - t11) * 4; }
  else { d[0] = descale(t10 + t11, 2); d[4 * s] = descale(t10 - t11, 2); }
  int z1 = (t12 + t13) * 4433;
  d[2 * s] = descale(z1 + t13 * 6270, sh);
  d[6 * s] = descale(z1 - t12 * 15137, sh);
  z1 = t4 + t7;
  int z2 = t5 + t6, z3 = t4 + t6, z4 = t5 + t7;
  const int z5 = (z3 + z4) * 9633;
  z1 *= -7373;
  z2 *= -20995;
  z3 = z3 * -16069 + z5;
  z4 = z4 * -3196 + z5;
  d[7 * s] = descale(t4 * 2446 + z1 + z3, sh);
  d[5 * s] = descale(t5 * 16819 + z2 + z4, sh);
  d[3 * s] = descale(t6 * 25172 + z2 + z3, sh);
  d[s] = descale(t7 * 12299 + z1 + z4, sh);
}

// one component sample: libjpeg's rgb_ycc_convert, then the downsampler jcsample.c picks for (he, ve)
__device__ __forceinline__ int component_sample(const EncImg& m, const uint8_t* src, int c, int cx, int cy, int he,
                                                int ve, int row_cap) {
  cy = min(cy, row_cap);
  int sum = 0;
  for (int dy = 0; dy < ve; ++dy) {
    const uint8_t* row = src + (int64_t)min(cy * ve + dy, m.H - 1) * m.pitch;
    for (int dx = 0; dx < he; ++dx) {
      const int x = min(cx * he + dx, m.W - 1);
      if (m.channels == 1) { sum += row[x]; continue; }
      const int b = row[3 * x], g = row[3 * x + 1], r = row[3 * x + 2];
      if (c == 0) sum += (19595 * r + 38470 * g + 7471 * b + 32768) >> 16;
      else if (c == 1) sum += (-11059 * r - 21709 * g + 32768 * b + (128 << 16) + 32767) >> 16;
      else sum += (32768 * r - 27439 * g - 5329 * b + (128 << 16) + 32767) >> 16;
    }
  }
  if (he == 1 && ve == 1) return sum;
  if (he == 2 && ve == 1) return (sum + (cx & 1)) >> 1;         // h2v1: bias 0, 1, 0, 1, ...
  if (he == 2 && ve == 2) return (sum + 1 + (cx & 1)) >> 2;     // h2v2: bias 1, 2, 1, 2, ...
  const int np = he * ve;                                       // generic integer downsampler
  return (sum + np / 2) / np;
}

__global__ void __launch_bounds__(kBlockThreads) enc_fdct(const uint8_t* __restrict__ blob, uint8_t* __restrict__ ws) {
  const EncBatch& B = *reinterpret_cast<const EncBatch*>(blob);
  const EncImg& m = enc_img(blob, blockIdx.y);
  const int64_t b = (int64_t)blockIdx.x * kBlockThreads + threadIdx.x;
  if (b >= m.nblocks) return;
  const int64_t mcu = b / m.bpm;
  const int k = (int)(b - mcu * m.bpm);
  const int mx = (int)(mcu % m.mcus_x), my = (int)(mcu / m.mcus_x);
  const int c = m.blk_comp[k], ch = m.ch[c], cv = m.cv[c];
  int bx = m.blk_x[k], by = m.blk_y[k];
  // a dummy block (past the component's own blocks) takes the DC of the block before it in its MCU, which chains
  // back to the last real block of its row, or of the last real row
  const int xv = min(ch, m.wib[c] - mx * ch), yv = min(cv, m.hib[c] - my * cv);
  const bool dummy = bx >= xv || by >= yv;
  if (by >= yv) { bx = xv - 1; by = yv - 1; }
  else if (bx >= xv) bx = xv - 1;
  const int gx = mx * ch + bx, gy = my * cv + by;
  const int he = m.hmax / ch, ve = m.vmax / cv;
  // component rows past the last row group of vmax image rows repeat that group's last component row
  const int row_cap = (m.H + m.vmax - 1) / m.vmax * cv - 1;
  const uint8_t* src = reinterpret_cast<const uint8_t*>(m.src);
  int d[64];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) d[8 * i + j] = component_sample(m, src, c, gx * 8 + j, gy * 8 + i, he, ve, row_cap) - 128;
#pragma unroll
  for (int i = 0; i < 8; ++i) fdct_1d<0>(d + 8 * i, 1);
#pragma unroll
  for (int j = 0; j < 8; ++j) fdct_1d<1>(d + j, 8);
  const int t = c ? 1 : 0;
  // a local copy: with the loop unrolled every index is a constant and d stays in registers
  constexpr uint8_t zz[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                              41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                              30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
  int16_t q[64];
#pragma unroll
  for (int z = 0; z < 64; ++z) {
    const int i = zz[z];
    const int x = d[i], a = x < 0 ? -x : x;
    const int v = (int)(((uint32_t)(a + m.corr[t][i]) * m.recip[t][i]) >> m.shift[t][i]);
    q[z] = (int16_t)(dummy && z ? 0 : (x < 0 ? -v : v));
  }
  int4* out = reinterpret_cast<int4*>(ws + B.ws_coef) + (m.blk_base + b) * 8;
  const int4* qv = reinterpret_cast<const int4*>(q);
#pragma unroll
  for (int v = 0; v < 8; ++v) out[v] = qv[v];
}

// The block whose DC predicts block b's (same component, previous in scan order, same restart segment), or -1.
__device__ __forceinline__ int64_t dc_pred_block(const EncImg& m, int64_t b) {
  const int64_t mcu = b / m.bpm;
  const int k = (int)(b - mcu * m.bpm);
  const int c = m.blk_comp[k];
  if (k > 0 && m.blk_comp[k - 1] == c) return b - 1;
  if (mcu == 0 || (m.ri && mcu % m.ri == 0)) return -1;
  int last = k;
  while (last + 1 < m.bpm && m.blk_comp[last + 1] == c) ++last;
  return (mcu - 1) * m.bpm + last;
}

__device__ __forceinline__ void load_block(const uint8_t* ws, const EncBatch& B, int64_t gb, int16_t (&q)[64]) {
  const int4* in = reinterpret_cast<const int4*>(ws + B.ws_coef) + gb * 8;
  int4* qv = reinterpret_cast<int4*>(q);
#pragma unroll
  for (int v = 0; v < 8; ++v) qv[v] = in[v];
}

__device__ __forceinline__ int nbits(int v) { return v ? 32 - __clz(v < 0 ? -v : v) : 0; }

// Walks block b's Huffman symbols: emit(code, length) for each code and each size field, in stream order.
template <typename Emit>
__device__ __forceinline__ void block_symbols(const int16_t (&q)[64], int dc_prev, const uint32_t* dc_code,
                                             const uint32_t* ac_code, Emit&& emit) {
  const int diff = q[0] - dc_prev;
  int s = nbits(diff);
  uint32_t e = dc_code[s];
  emit(e >> 8, (int)(e & 255));
  if (s) emit((uint32_t)(diff < 0 ? diff - 1 : diff) & ((1u << s) - 1), s);
  int run = 0;
  for (int k = 1; k < 64; ++k) {
    const int v = q[k];
    if (v == 0) { ++run; continue; }
    for (; run > 15; run -= 16) { e = ac_code[0xF0]; emit(e >> 8, (int)(e & 255)); }
    s = nbits(v);
    e = ac_code[run << 4 | s];
    emit(e >> 8, (int)(e & 255));
    emit((uint32_t)(v < 0 ? v - 1 : v) & ((1u << s) - 1), s);
    run = 0;
  }
  if (run) { e = ac_code[0]; emit(e >> 8, (int)(e & 255)); }
}

__device__ __forceinline__ void load_codes(const EncBatch& B, uint32_t* s_dc, uint32_t* s_ac) {
  for (int i = threadIdx.x; i < 2 * 16; i += blockDim.x) s_dc[i] = (&B.dc_code[0][0])[i];
  for (int i = threadIdx.x; i < 2 * 256; i += blockDim.x) s_ac[i] = (&B.ac_code[0][0])[i];
  __syncthreads();
}

__device__ __forceinline__ int block_dc_prev(const uint8_t* ws, const EncBatch& B, const EncImg& m, int64_t b) {
  const int64_t p = dc_pred_block(m, b);
  return p < 0 ? 0 : reinterpret_cast<const int16_t*>(ws + B.ws_coef)[(m.blk_base + p) * 64];
}

__global__ void __launch_bounds__(kBlockThreads) enc_count(const uint8_t* __restrict__ blob, uint8_t* __restrict__ ws) {
  __shared__ uint32_t s_dc[2 * 16], s_ac[2 * 256];
  const EncBatch& B = *reinterpret_cast<const EncBatch*>(blob);
  load_codes(B, s_dc, s_ac);
  const EncImg& m = enc_img(blob, blockIdx.y);
  const int64_t b = (int64_t)blockIdx.x * kBlockThreads + threadIdx.x;
  if (b >= m.nblocks) return;
  int16_t q[64];
  load_block(ws, B, m.blk_base + b, q);
  const int t = m.blk_comp[b % m.bpm] ? 1 : 0;
  uint32_t bits = 0;
  block_symbols(q, block_dc_prev(ws, B, m, b), s_dc + 16 * t, s_ac + 256 * t, [&](uint32_t, int len) { bits += len; });
  reinterpret_cast<uint32_t*>(ws + B.ws_bits)[m.blk_base + b] = bits;
  const int64_t seg = m.ri ? b / m.bpm / m.ri : 0;
  atomicAdd(reinterpret_cast<unsigned long long*>(ws + B.ws_seg_bits) + m.seg_base + seg, (unsigned long long)bits);
}

// Block-wide segmented inclusive scan over (flag, value): a flagged element starts a new sum.  carry is the sum of
// the segment still open at the end of the previous call; it is updated for the next call.
__device__ uint64_t block_seg_scan(bool flag, uint64_t v, uint64_t& carry, uint64_t* s_v, int* s_f) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  int f = flag;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint64_t uv = __shfl_up_sync(0xffffffffu, v, d);
    const int uf = __shfl_up_sync(0xffffffffu, f, d);
    if (lane >= d) { if (!f) v += uv; f |= uf; }
  }
  if (lane == 31) { s_v[warp] = v; s_f[warp] = f; }
  __syncthreads();
  if (warp == 0) {
    uint64_t wv = lane < nw ? s_v[lane] : 0;
    int wf = lane < nw ? s_f[lane] : 0;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const uint64_t uv = __shfl_up_sync(0xffffffffu, wv, d);
      const int uf = __shfl_up_sync(0xffffffffu, wf, d);
      if (lane >= d) { if (!wf) wv += uv; wf |= uf; }
    }
    if (!wf) wv += carry;          // inclusive over warps, with the carry folded in
    if (lane < nw) s_v[32 + lane] = wv;
  }
  __syncthreads();
  if (!f) v += warp ? s_v[32 + warp - 1] : carry;
  const uint64_t next = s_v[32 + nw - 1];
  __syncthreads();
  carry = next;
  return v;
}

__global__ void __launch_bounds__(kScanThreads) enc_scan(const uint8_t* __restrict__ blob, uint8_t* __restrict__ ws) {
  __shared__ uint64_t s_v[64];
  __shared__ int s_f[32];
  const EncBatch& B = *reinterpret_cast<const EncBatch*>(blob);
  const EncImg& m = enc_img(blob, blockIdx.x);
  const uint64_t* seg_bits = reinterpret_cast<const uint64_t*>(ws + B.ws_seg_bits) + m.seg_base;
  uint64_t* seg_start = reinterpret_cast<uint64_t*>(ws + B.ws_seg_start) + m.seg_base;
  uint64_t carry = 0;
  for (int64_t s0 = 0; s0 < m.nseg; s0 += kScanThreads) {      // segment starts, each on a chunk
    const int64_t s = s0 + threadIdx.x;
    const uint64_t len = s < m.nseg ? (seg_bits[s] + kChunkBits - 1) / kChunkBits * kChunkBits : 0;
    const uint64_t incl = block_seg_scan(false, len, carry, s_v, s_f);
    if (s < m.nseg) seg_start[s] = incl - len;
  }
  const uint64_t used_words = carry / 32;
  __syncthreads();
  const uint32_t* bits = reinterpret_cast<const uint32_t*>(ws + B.ws_bits) + m.blk_base;
  uint64_t* off = reinterpret_cast<uint64_t*>(ws + B.ws_off) + m.blk_base;
  const int64_t seg_blocks = m.ri ? (int64_t)m.ri * m.bpm : m.nblocks;
  carry = 0;
  for (int64_t b0 = 0; b0 < m.nblocks; b0 += kScanThreads) {   // block offsets within their segment
    const int64_t b = b0 + threadIdx.x;
    const uint64_t v = b < m.nblocks ? bits[b] : 0;
    const uint64_t incl = block_seg_scan(b < m.nblocks && b % seg_blocks == 0, v, carry, s_v, s_f);
    if (b < m.nblocks) off[b] = seg_start[b / seg_blocks] + incl - v;
  }
  uint32_t* words = reinterpret_cast<uint32_t*>(ws + B.ws_words) + m.word_base;
  for (uint64_t w = threadIdx.x; w < used_words; w += kScanThreads) words[w] = 0;
  if (threadIdx.x == 0) reinterpret_cast<int64_t*>(ws + B.ws_img)[2 * blockIdx.x] = (int64_t)(used_words / 32);
}

__global__ void __launch_bounds__(kBlockThreads) enc_emit(const uint8_t* __restrict__ blob, uint8_t* __restrict__ ws) {
  __shared__ uint32_t s_dc[2 * 16], s_ac[2 * 256];
  const EncBatch& B = *reinterpret_cast<const EncBatch*>(blob);
  load_codes(B, s_dc, s_ac);
  const EncImg& m = enc_img(blob, blockIdx.y);
  const int64_t b = (int64_t)blockIdx.x * kBlockThreads + threadIdx.x;
  if (b >= m.nblocks) return;
  int16_t q[64];
  load_block(ws, B, m.blk_base + b, q);
  const int t = m.blk_comp[b % m.bpm] ? 1 : 0;
  const uint64_t start = reinterpret_cast<const uint64_t*>(ws + B.ws_off)[m.blk_base + b];
  uint32_t* words = reinterpret_cast<uint32_t*>(ws + B.ws_words) + m.word_base;
  uint64_t w = start >> 5;
  uint64_t acc = 0;
  int nacc = (int)(start & 31);       // bits of the current word before this block's
  auto put = [&](uint32_t code, int len) {
    acc = acc << len | code;
    nacc += len;
    if (nacc >= 32) {
      nacc -= 32;
      atomicOr(words + w++, (uint32_t)(acc >> nacc));
      acc &= (1ull << nacc) - 1;
    }
  };
  block_symbols(q, block_dc_prev(ws, B, m, b), s_dc + 16 * t, s_ac + 256 * t, put);
  const int64_t seg_blocks = m.ri ? (int64_t)m.ri * m.bpm : m.nblocks;
  if ((b + 1) % seg_blocks == 0 || b + 1 == m.nblocks) {        // pad the segment to a byte with 1-bits
    const int pad = (8 - (nacc & 7)) & 7;
    if (pad) put((1u << pad) - 1, pad);
  }
  if (nacc) atomicOr(words + w, (uint32_t)(acc << (32 - nacc)));
}

__device__ __forceinline__ int ff_bytes(uint32_t w) {
  int n = 0;
#pragma unroll
  for (int j = 0; j < 4; ++j) n += ((w >> (8 * j)) & 255) == 255;
  return n;
}

// segment of chunk c: the last segment starting at or before it
__device__ __forceinline__ int64_t chunk_segment(const uint64_t* seg_start, int64_t nseg, int64_t c) {
  int64_t lo = 0, hi = nseg - 1;
  const uint64_t bit = (uint64_t)c * kChunkBits;
  while (lo < hi) {
    const int64_t mid = (lo + hi + 1) / 2;
    if (seg_start[mid] <= bit) lo = mid; else hi = mid - 1;
  }
  return lo;
}

__global__ void __launch_bounds__(256) enc_ffcount(const uint8_t* __restrict__ blob, uint8_t* __restrict__ ws) {
  const EncBatch& B = *reinterpret_cast<const EncBatch*>(blob);
  const EncImg& m = enc_img(blob, blockIdx.y);
  const int64_t used = reinterpret_cast<const int64_t*>(ws + B.ws_img)[2 * blockIdx.y];
  const uint64_t* seg_start = reinterpret_cast<const uint64_t*>(ws + B.ws_seg_start) + m.seg_base;
  const uint32_t* words = reinterpret_cast<const uint32_t*>(ws + B.ws_words) + m.word_base;
  const int lane = threadIdx.x & 31;
  for (int64_t c = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5); c < used; c += (int64_t)gridDim.x * 8) {
    int n = ff_bytes(words[c * 32 + lane]);
#pragma unroll
    for (int d = 16; d; d >>= 1) n += __shfl_xor_sync(0xffffffffu, n, d);
    if (lane == 0) {
      const int64_t s = chunk_segment(seg_start, m.nseg, c);
      const bool first = seg_start[s] == (uint64_t)c * kChunkBits;
      reinterpret_cast<uint32_t*>(ws + B.ws_chunk_ff)[m.chunk_base + c] = (uint32_t)n;
      reinterpret_cast<uint32_t*>(ws + B.ws_chunk_seg)[m.chunk_base + c] = (uint32_t)s | (first ? 0x80000000u : 0u);
      if (n) atomicAdd(reinterpret_cast<unsigned long long*>(ws + B.ws_seg_ff) + m.seg_base + s, (unsigned long long)n);
    }
  }
}

__global__ void __launch_bounds__(kScanThreads) enc_layout(const uint8_t* __restrict__ blob, uint8_t* __restrict__ ws) {
  __shared__ uint64_t s_v[64];
  __shared__ int s_f[32];
  const EncBatch& B = *reinterpret_cast<const EncBatch*>(blob);
  const EncImg& m = enc_img(blob, blockIdx.x);
  int64_t* img = reinterpret_cast<int64_t*>(ws + B.ws_img) + 2 * blockIdx.x;
  const int64_t used = img[0];
  const uint32_t* cff = reinterpret_cast<const uint32_t*>(ws + B.ws_chunk_ff) + m.chunk_base;
  const uint32_t* cseg = reinterpret_cast<const uint32_t*>(ws + B.ws_chunk_seg) + m.chunk_base;
  uint64_t* before = reinterpret_cast<uint64_t*>(ws + B.ws_chunk_before) + m.chunk_base;
  uint64_t carry = 0;
  for (int64_t c0 = 0; c0 < used; c0 += kScanThreads) {        // 0xFF bytes before each chunk in its segment
    const int64_t c = c0 + threadIdx.x;
    const uint64_t v = c < used ? cff[c] : 0;
    const uint64_t incl = block_seg_scan(c < used && (cseg[c] >> 31), v, carry, s_v, s_f);
    if (c < used) before[c] = incl - v;
  }
  const uint64_t* seg_bits = reinterpret_cast<const uint64_t*>(ws + B.ws_seg_bits) + m.seg_base;
  const uint64_t* seg_ff = reinterpret_cast<const uint64_t*>(ws + B.ws_seg_ff) + m.seg_base;
  uint64_t* seg_out = reinterpret_cast<uint64_t*>(ws + B.ws_seg_out) + m.seg_base;
  carry = 0;
  for (int64_t s0 = 0; s0 < m.nseg; s0 += kScanThreads) {      // stuffed segments, each after its RSTn
    const int64_t s = s0 + threadIdx.x;
    const uint64_t v = s < m.nseg ? (seg_bits[s] + 7) / 8 + seg_ff[s] + (s ? 2 : 0) : 0;
    const uint64_t incl = block_seg_scan(false, v, carry, s_v, s_f);
    if (s < m.nseg) seg_out[s] = incl - v;
  }
  if (threadIdx.x == 0) img[1] = m.hdr_len + (int64_t)carry + 2;
}

__global__ void __launch_bounds__(kScanThreads) enc_files(const uint8_t* __restrict__ blob, uint8_t* __restrict__ ws,
                                                          int64_t* __restrict__ out_desc) {
  __shared__ uint64_t s_v[64];
  __shared__ int s_f[32];
  const EncBatch& B = *reinterpret_cast<const EncBatch*>(blob);
  const int64_t* img = reinterpret_cast<const int64_t*>(ws + B.ws_img);
  uint64_t carry = 0;
  for (int i0 = 0; i0 < B.n; i0 += kScanThreads) {
    const int i = i0 + threadIdx.x;
    const uint64_t v = i < B.n ? (uint64_t)img[2 * i + 1] : 0;
    const uint64_t incl = block_seg_scan(false, v, carry, s_v, s_f);
    if (i < B.n) { out_desc[2 * i] = (int64_t)(incl - v); out_desc[2 * i + 1] = (int64_t)v; }
  }
}

__global__ void __launch_bounds__(256) enc_assemble(const uint8_t* __restrict__ blob, const uint8_t* __restrict__ ws,
                                                    const int64_t* __restrict__ out_desc, uint8_t* __restrict__ out) {
  const EncBatch& B = *reinterpret_cast<const EncBatch*>(blob);
  const EncImg& m = enc_img(blob, blockIdx.y);
  uint8_t* file = out + out_desc[2 * blockIdx.y];
  if (blockIdx.x == 0) {
    for (int i = threadIdx.x; i < m.hdr_len; i += blockDim.x) file[i] = blob[m.hdr_off + i];
    if (threadIdx.x == 0) {
      const int64_t len = out_desc[2 * blockIdx.y + 1];
      file[len - 2] = 0xFF;
      file[len - 1] = 0xD9;
    }
  }
  const int64_t used = reinterpret_cast<const int64_t*>(ws + B.ws_img)[2 * blockIdx.y];
  const uint64_t* seg_start = reinterpret_cast<const uint64_t*>(ws + B.ws_seg_start) + m.seg_base;
  const uint64_t* seg_bits = reinterpret_cast<const uint64_t*>(ws + B.ws_seg_bits) + m.seg_base;
  const uint64_t* seg_out = reinterpret_cast<const uint64_t*>(ws + B.ws_seg_out) + m.seg_base;
  const uint32_t* cseg = reinterpret_cast<const uint32_t*>(ws + B.ws_chunk_seg) + m.chunk_base;
  const uint64_t* before = reinterpret_cast<const uint64_t*>(ws + B.ws_chunk_before) + m.chunk_base;
  const uint32_t* words = reinterpret_cast<const uint32_t*>(ws + B.ws_words) + m.word_base;
  const int lane = threadIdx.x & 31;
  uint8_t* data = file + m.hdr_len;
  for (int64_t c = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5); c < used; c += (int64_t)gridDim.x * 8) {
    const int64_t s = cseg[c] & 0x7fffffffu;
    const uint64_t first = seg_start[s] / kChunkBits, nbytes = (seg_bits[s] + 7) / 8;
    const uint64_t byte0 = (c - first) * (kChunkBits / 8) + 4 * lane;    // of this lane's word in the segment
    const uint32_t w = words[c * 32 + lane];
    uint8_t v[4];
    int nv = 0, ff = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      v[j] = (uint8_t)(w >> (24 - 8 * j));
      if (byte0 + j < nbytes) { ++nv; ff += v[j] == 255; }
    }
    int incl = ff;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int u = __shfl_up_sync(0xffffffffu, incl, d);
      if (lane >= d) incl += u;
    }
    uint8_t* seg = data + seg_out[s];
    if (s && c == (int64_t)first && lane == 0) { seg[0] = 0xFF; seg[1] = (uint8_t)(0xD0 + ((s - 1) & 7)); }
    uint8_t* o = seg + (s ? 2 : 0) + byte0 + before[c] + (incl - ff);
    for (int j = 0; j < nv; ++j) {
      *o++ = v[j];
      if (v[j] == 255) *o++ = 0;
    }
  }
}

}  // namespace
}  // namespace yb

using namespace yb;

extern "C" int yb_jpeg_enc_header(const yb_jpeg_enc_image* image, uint8_t* out, size_t capacity, size_t* bytes) {
  YB_REQUIRE(image && bytes, "yb_jpeg_enc_header: null argument");
  Resolved R;
  const int rc = resolve(*image, R);
  if (rc) return rc;
  uint8_t h[kMaxHeader];
  const size_t len = build_header(*image, R, h);
  *bytes = len;
  if (!out) return YB_OK;
  if (capacity < len) {
    set_error("yb_jpeg_enc_header: capacity %zu, %zu needed", capacity, len);
    return YB_ERR_WORKSPACE;
  }
  memcpy(out, h, len);
  return YB_OK;
}

extern "C" int yb_jpeg_enc_pack_bytes(const yb_jpeg_enc_image* images, int n, size_t* blob_bytes) {
  YB_REQUIRE(blob_bytes, "yb_jpeg_enc_pack_bytes: null blob_bytes");
  EncPlan P;
  const int rc = plan_enc(images, n, P);
  if (rc) return rc;
  *blob_bytes = (size_t)P.blob_bytes;
  return YB_OK;
}

extern "C" int yb_jpeg_enc_pack(const yb_jpeg_enc_image* images, int n, void* host_blob, size_t blob_bytes) {
  YB_REQUIRE(host_blob, "yb_jpeg_enc_pack: null host_blob");
  EncPlan P;
  const int rc = plan_enc(images, n, P);
  if (rc) return rc;
  YB_REQUIRE((int64_t)blob_bytes >= P.blob_bytes, "yb_jpeg_enc_pack: blob of %zu bytes, %lld needed", blob_bytes,
             (long long)P.blob_bytes);
  uint8_t* o = static_cast<uint8_t*>(host_blob);
  memset(o, 0, (size_t)P.blob_bytes);
  memcpy(o, &P.B, sizeof(EncBatch));
  memcpy(o + sizeof(EncBatch), P.img.data(), sizeof(EncImg) * (size_t)n);
  if (!P.hdr.empty()) memcpy(o + P.img[0].hdr_off, P.hdr.data(), P.hdr.size());
  return YB_OK;
}

extern "C" int yb_jpeg_enc_workspace_bytes(const void* host_blob, int n, size_t* workspace_bytes, size_t* out_bytes) {
  const EncBatch* B;
  const int rc = check_enc_blob(host_blob, n, B);
  if (rc) return rc;
  YB_REQUIRE(workspace_bytes, "yb_jpeg_enc_workspace_bytes: null workspace_bytes");
  *workspace_bytes = (size_t)B->ws_bytes;
  if (out_bytes) *out_bytes = (size_t)B->out_bytes;
  return YB_OK;
}

extern "C" int yb_jpeg_enc_encode(const void* dev_blob, const void* host_blob, int n, uint8_t* out, size_t out_bytes,
                                  int64_t* out_desc, void* workspace, size_t workspace_bytes, void* stream) {
  const EncBatch* B;
  const int rc = check_enc_blob(host_blob, n, B);
  if (rc) return rc;
  YB_REQUIRE(dev_blob && out && out_desc, "yb_jpeg_enc_encode: null device pointer");
  YB_REQUIRE(workspace, "yb_jpeg_enc_encode: null workspace");
  YB_REQUIRE((int64_t)out_bytes >= B->out_bytes, "yb_jpeg_enc_encode: output of %zu bytes, %lld needed", out_bytes,
             (long long)B->out_bytes);
  if (workspace_bytes < (size_t)B->ws_bytes) {
    set_error("yb_jpeg_enc_encode: workspace of %zu bytes, %lld needed", workspace_bytes, (long long)B->ws_bytes);
    return YB_ERR_WORKSPACE;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const uint8_t* blob = static_cast<const uint8_t*>(dev_blob);
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  YB_CUDA(cudaMemsetAsync(ws + B->ws_seg_bits, 0, (size_t)(16 * B->total_segs), st));   // seg_bits, seg_ff
  const dim3 blocks_grid((unsigned)((B->max_blocks + kBlockThreads - 1) / kBlockThreads), (unsigned)n);
  const dim3 chunk_grid((unsigned)std::min<int64_t>((B->max_chunks + 7) / 8, 64), (unsigned)n);
  enc_fdct<<<blocks_grid, kBlockThreads, 0, st>>>(blob, ws);
  YB_CUDA(cudaGetLastError());
  enc_count<<<blocks_grid, kBlockThreads, 0, st>>>(blob, ws);
  YB_CUDA(cudaGetLastError());
  enc_scan<<<n, kScanThreads, 0, st>>>(blob, ws);
  YB_CUDA(cudaGetLastError());
  enc_emit<<<blocks_grid, kBlockThreads, 0, st>>>(blob, ws);
  YB_CUDA(cudaGetLastError());
  enc_ffcount<<<chunk_grid, 256, 0, st>>>(blob, ws);
  YB_CUDA(cudaGetLastError());
  enc_layout<<<n, kScanThreads, 0, st>>>(blob, ws);
  YB_CUDA(cudaGetLastError());
  enc_files<<<1, kScanThreads, 0, st>>>(blob, ws, out_desc);
  YB_CUDA(cudaGetLastError());
  enc_assemble<<<chunk_grid, 256, 0, st>>>(blob, ws, out_desc, out);
  YB_CUDA(cudaGetLastError());
  return YB_OK;
}
