// Detection drawing on the device: the reference's plot_one_box (utils/plot_utils.py) over a whole batch, equal
// to OpenCV 4.13's pixels bit for bit.  Per detection, in NMS order: cv2.rectangle(c1, c2, color, tl) with LINE_8,
// the filled label rectangle, and cv2.putText(label, FONT_HERSHEY_SIMPLEX, tl / 3, black, max(tl - 1, 1), LINE_AA).
//
// Pixel-owner rasterisation: a CTA owns a 32 x 32 tile of one image and each thread four of its pixels, held in
// registers.  The CTA walks the image's detections in order; for every primitive that can reach the tile, each
// thread applies it to its own pixels with a closed form of OpenCV's incremental stepping.  A pixel therefore sees
// the same sequence of writes and blends as under OpenCV, and no two threads share a pixel.
//
// The closed forms (DESIGN.md §4 has the argument):
// - rectangle outline, one colour: a set.  tl <= 1 is four axis-parallel 1-pixel lines.  tl >= 2 is, per side,
//   ThickLine's quad, whose corners are whole pixels because an axis-parallel side's offset is (tl + (tl & 1)) / 2
//   exactly; plus the midpoint circle Circle(corner, (tl + 1) >> 1) filled at each corner.
// - filled rectangle: the clipped box.
// - LineAA: step k of the major axis sits at start + k, with the minor coordinate minor0 + k * step (OpenCV adds
//   step k times; the sum is exact in int64) and the end-point correction picked from (k, steps - k).  Clipping is
//   OpenCV's clipLine in double, done once per segment by every thread alike.
// - thick text (font thickness >= 2): ThickLine's quad and round caps, each FillConvexPoly with LINE_AA: LineAA
//   along its edges, then OpenCV's scanline edge walk, replayed row by row by every thread alike.
#include <math.h>
#include <string.h>

#include "common.cuh"
#include "hershey_simplex.inc"

namespace {

constexpr int kTile = 32;
constexpr int kThreads = 256;
constexpr int kPix = kTile * kTile / kThreads;           // 4 pixels per thread: one column, rows r, r + 8, ...
constexpr int kMaxTl = 1023;
constexpr float kCoordClamp = 16777216.f;                // 2^24: see yb_plot_boxes in yolob200.h
constexpr int kHeaderWords = 4;

#define YB_GLYPH_INIT YB_HS_GLYPHS
__constant__ char c_glyphs[] = YB_GLYPH_INIT;
__constant__ unsigned short c_glyph_off[96] = YB_HS_GLYPH_OFFSETS;
__constant__ int c_filter[64] = YB_AA_FILTER;
__constant__ int c_slope_corr[32] = YB_AA_SLOPE_CORR;
__constant__ float c_sin[451] = YB_SIN_TABLE;
[[maybe_unused]] static const char h_glyphs[] = YB_GLYPH_INIT;
[[maybe_unused]] static const unsigned short h_glyph_off[96] = YB_HS_GLYPH_OFFSETS;

__host__ __device__ inline const char* glyph(int code) {
#ifdef __CUDA_ARCH__
  return c_glyphs + c_glyph_off[code - 32];
#else
  return h_glyphs + h_glyph_off[code - 32];
#endif
}

// double arithmetic without contraction, so host and device round alike
__host__ __device__ inline double dmul(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}
__host__ __device__ inline double dadd(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}
__host__ __device__ inline int cv_round(double v) {       // cvRound: nearest, ties to even
#ifdef __CUDA_ARCH__
  return __double2int_rn(v);
#else
  return (int)nearbyint(v);
#endif
}

// putText / getTextSize read FONT_HERSHEY_SIMPLEX text byte by byte; bytes outside ' ' .. '~' draw '?'
__host__ __device__ inline int text_code(unsigned char b) { return b >= 32 && b < 127 ? b : '?'; }

// '{:.2f}'.format(np.float32(score) * 100): the float32 product rounded to two decimals exactly, ties to even
// (Python formats the exact binary value), with the reference's ", " before and "%" after.
__host__ __device__ __noinline__ int format_score(float score, unsigned char* out) {
  int n = 0;
  out[n++] = ',';
  out[n++] = ' ';
#ifdef __CUDA_ARCH__
  const float v = __fmul_rn(score, 100.f);
#else
  const float v = score * 100.f;
#endif
  uint32_t bits;
  memcpy(&bits, &v, 4);
  const bool neg = bits >> 31;
  const uint32_t ex = (bits >> 23) & 255, fr = bits & 0x7fffff;
  if (ex == 255 && fr) {                                   // Python prints every NaN as "nan"
    out[n++] = 'n'; out[n++] = 'a'; out[n++] = 'n'; out[n++] = '%';
    return n;
  }
  if (neg) out[n++] = '-';
  if (ex == 255) {
    out[n++] = 'i'; out[n++] = 'n'; out[n++] = 'f'; out[n++] = '%';
    return n;
  }
  const uint64_t m = ex ? (fr | 0x800000u) : fr;           // |v| = m * 2^e
  const int e = ex ? (int)ex - 150 : -149;
  unsigned __int128 ip;                                    // integer part
  uint32_t cents;
  if (e >= 0) {
    ip = (unsigned __int128)m << e;
    cents = 0;
  } else {
    const int k = -e;                                      // 100 |v| = (100 m) / 2^k, rounded half to even
    const uint64_t num = m * 100;
    uint64_t q = 0;
    if (k < 63) {
      q = num >> k;
      const uint64_t r = num - (q << k), half = 1ull << (k - 1);
      if (r > half || (r == half && (q & 1))) q++;
    }                                                      // k >= 63: 100 m < 2^31 is below half an ulp of 0.01
    ip = q / 100;
    cents = (uint32_t)(q % 100);
  }
  unsigned char digits[40];
  int nd = 0;
  do {
    digits[nd++] = (unsigned char)('0' + (int)(ip % 10));
    ip /= 10;
  } while (ip);
  while (nd) out[n++] = digits[--nd];
  out[n++] = '.';
  out[n++] = (unsigned char)('0' + cents / 10);
  out[n++] = (unsigned char)('0' + cents % 10);
  out[n++] = '%';
  return n;
}

// The label of one detection: text codes, getTextSize and the reference's rectangle and text origin.
__host__ __device__ void label_layout(const unsigned char* name, int name_len, int with_score, float score, int tl,
                                      int x0, int y0, unsigned char* text, yb_plot_layout* L) {
  int len = 0;
  for (int i = 0; i < name_len; i++) text[len++] = (unsigned char)text_code(name[i]);
  if (with_score) len += format_score(score, text + len);
  const int tf = tl - 1 > 1 ? tl - 1 : 1;
  const double scale = (double)tl / 3.0;
  double view_x = 0.0;
  for (int i = 0; i < len; i++) {
    const char* g = glyph(text[i]);
    view_x = dadd(view_x, dmul((double)(g[1] - g[0]), scale));
  }
  L->length = len;
  L->thickness = tf;
  L->text_w = cv_round(dadd(view_x, (double)tf));
  L->text_h = cv_round(dadd(dmul((double)(YB_HS_CAP_LINE + YB_HS_BASE_LINE), scale), (double)((tf + 1) / 2)));
  L->rect_x1 = x0 + L->text_w;
  L->rect_y1 = y0 - L->text_h - 3;
  L->org_x = x0;
  L->org_y = y0 - 2;
}

// ---------------------------------------------------------------------------------------------------------------
// device drawing
// ---------------------------------------------------------------------------------------------------------------
struct Px {                                                // a thread's pixels
  int x, y[kPix];
  int v[kPix][3];
  bool in[kPix];
};

__device__ inline void set_rect(Px& p, int xa, int ya, int xb, int yb, const int* col) {
  const int x0 = min(xa, xb), x1 = max(xa, xb), y0 = min(ya, yb), y1 = max(ya, yb);
  if (p.x < x0 || p.x > x1) return;
#pragma unroll
  for (int k = 0; k < kPix; k++)
    if (p.y[k] >= y0 && p.y[k] <= y1) { p.v[k][0] = col[0]; p.v[k][1] = col[1]; p.v[k][2] = col[2]; }
}

// cv2.rectangle(c1, c2, col, tl), LINE_8: a set of pixels of one colour (see the file comment)
__device__ void outline(Px& p, int x0, int y0, int x1, int y1, int tl, const int* col, const int* spans) {
  if (tl <= 1) {
    set_rect(p, x0, y0, x1, y0, col);
    set_rect(p, x0, y1, x1, y1, col);
    set_rect(p, x0, y0, x0, y1, col);
    set_rect(p, x1, y0, x1, y1, col);
    return;
  }
  const int h = (tl + 1) / 2, r = (tl + 1) >> 1;
  if (x0 != x1) {
    set_rect(p, x0, y0 - h, x1, y0 + h, col);
    set_rect(p, x0, y1 - h, x1, y1 + h, col);
  }
  if (y0 != y1) {
    set_rect(p, x0 - h, y0, x0 + h, y1, col);
    set_rect(p, x1 - h, y0, x1 + h, y1, col);
  }
  const int cx[2] = {x0, x1}, cy[2] = {y0, y1};
#pragma unroll
  for (int k = 0; k < kPix; k++)
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const int dx = abs(p.x - cx[i & 1]), dy = abs(p.y[k] - cy[i >> 1]);
      if (dy <= r && dx <= spans[dy]) { p.v[k][0] = col[0]; p.v[k][1] = col[1]; p.v[k][2] = col[2]; }
    }
}

// OpenCV's clipLine (Size2l, Point2l)
__device__ bool clip_line(int64_t w, int64_t h, int64_t& x1, int64_t& y1, int64_t& x2, int64_t& y2) {
  const int64_t right = w - 1, bottom = h - 1;
  int c1 = (x1 < 0) + (x1 > right) * 2 + (y1 < 0) * 4 + (y1 > bottom) * 8;
  int c2 = (x2 < 0) + (x2 > right) * 2 + (y2 < 0) * 4 + (y2 > bottom) * 8;
  if ((c1 & c2) == 0 && (c1 | c2) != 0) {
    int64_t a;
    if (c1 & 12) {
      a = c1 < 8 ? 0 : bottom;
      x1 += (int64_t)(__ddiv_rn(__dmul_rn((double)(a - y1), (double)(x2 - x1)), (double)(y2 - y1)));
      y1 = a;
      c1 = (x1 < 0) + (x1 > right) * 2;
    }
    if (c2 & 12) {
      a = c2 < 8 ? 0 : bottom;
      x2 += (int64_t)(__ddiv_rn(__dmul_rn((double)(a - y2), (double)(x2 - x1)), (double)(y2 - y1)));
      y2 = a;
      c2 = (x2 < 0) + (x2 > right) * 2;
    }
    if ((c1 & c2) == 0 && (c1 | c2) != 0) {
      if (c1) {
        a = c1 == 1 ? 0 : right;
        y1 += (int64_t)(__ddiv_rn(__dmul_rn((double)(a - x1), (double)(y2 - y1)), (double)(x2 - x1)));
        x1 = a;
        c1 = 0;
      }
      if (c2) {
        a = c2 == 1 ? 0 : right;
        y2 += (int64_t)(__ddiv_rn(__dmul_rn((double)(a - x2), (double)(y2 - y1)), (double)(x2 - x1)));
        x2 = a;
        c2 = 0;
      }
    }
  }
  return (c1 | c2) == 0;
}

__device__ inline void blend_black(int* v, int a) {         // LineAA's put, which steps twice towards the colour
#pragma unroll
  for (int c = 0; c < 3; c++) {
    int t = v[c];
    t += (-t * a + 127) >> 8;
    t += (-t * a + 127) >> 8;
    v[c] = t;
  }
}

// LineAA(pt1, pt2) in black on this thread's pixels, 16.16 fixed-point end points
__device__ void line_aa(Px& p, int w, int h, int64_t x1, int64_t y1, int64_t x2, int64_t y2) {
  constexpr int S = 16;
  constexpr int64_t ONE = 1 << S;
  if (!clip_line((int64_t)w << S, (int64_t)h << S, x1, y1, x2, y2)) return;
  int64_t dx = x2 - x1, dy = y2 - y1;
  const int64_t ax = dx < 0 ? -dx : dx, ay = dy < 0 ? -dy : dy;
  const bool xmaj = ax > ay;
  int64_t step, start, minor, i, j;
  int ecount;
  if (xmaj) {
    if (dx < 0) { int64_t t = x1; x1 = x2; x2 = t; t = y1; y1 = y2; y2 = t; dy = -dy; }
    step = (dy * ONE) / (ax | 1);
    x2 += ONE;
    ecount = (int)((x2 >> S) - (x1 >> S));
    j = -(x1 & (ONE - 1));
    y1 += ((step * j) >> S) + (ONE >> 1);
    i = (x1 >> (S - 7)) & 0x78;
    j = (x2 >> (S - 7)) & 0x78;
    start = x1 >> S;
    minor = y1;
  } else {
    if (dy < 0) { int64_t t = x1; x1 = x2; x2 = t; t = y1; y1 = y2; y2 = t; dx = -dx; }
    step = (dx * ONE) / (ay | 1);
    y2 += ONE;
    ecount = (int)((y2 >> S) - (y1 >> S));
    j = -(y1 & (ONE - 1));
    x1 += ((step * j) >> S) + (ONE >> 1);
    i = (y1 >> (S - 7)) & 0x78;
    j = (y2 >> (S - 7)) & 0x78;
    start = y1 >> S;
    minor = x1;
  }
  int slope = (int)((step >> (S - 5)) & 0x3f);
  slope ^= step < 0 ? 0x3f : 0;
  slope = (slope & 0x20) ? 0x100 : c_slope_corr[slope];
  const int ii = (int)i, jj = (int)j;
  const int t0 = slope << 7, t1 = ((0x78 - ii) | 4) * slope, t2 = (jj | 4) * slope;
  int ep[9];
  ep[0] = 0;
  ep[8] = slope;
  ep[1] = ep[3] = ((((jj - ii) & 0x78) | 4) * slope >> 8) & 0x1ff;
  ep[2] = (t1 >> 8) & 0x1ff;
  ep[4] = ((((jj - ii) + 0x80) | 4) * slope >> 8) & 0x1ff;
  ep[5] = ((t1 + t0) >> 8) & 0x1ff;
  ep[6] = (t2 >> 8) & 0x1ff;
  ep[7] = ((t2 + t0) >> 8) & 0x1ff;
#pragma unroll
  for (int k = 0; k < kPix; k++) {
    if (!p.in[k]) continue;
    const int64_t maj = xmaj ? p.x : p.y[k], mnr = xmaj ? p.y[k] : p.x;
    const int64_t s = maj - start;                         // step index
    if (s < 0 || s > ecount) continue;
    const int64_t pos = minor + s * step;
    const int64_t d = mnr - ((pos >> S) - 1);
    if (d < 0 || d > 2) continue;
    const int sc = (int)s, ec = ecount - sc;
    const int e = (((sc >= 2) + 1) & (sc | 2)) * 3 + (((ec >= 2) + 1) & (ec | 2));
    int corr = 0;
#pragma unroll
    for (int q = 0; q < 9; q++) corr = q == e ? ep[q] : corr;       // a select keeps ep in registers
    const int dist = (int)((pos >> (S - 5)) & 31);
    const int f = c_filter[d == 0 ? dist + 32 : d == 1 ? dist : 63 - dist];
    blend_black(p.v[k], (corr * f >> 8) & 0xff);
  }
}

// A convex polygon's vertex k (16.16): ThickLine's quad, kept in registers
struct QuadPoly {
  int64_t x[4], y[4];
  static constexpr int n = 4;
  __device__ void at(int k, int64_t& px, int64_t& py) const {
    px = x[0];
    py = y[0];
#pragma unroll
    for (int q = 1; q < 4; q++)
      if (q == k) { px = x[q]; py = y[q]; }
  }
};

// EllipseEx(center, (r, r), 0, 0, 360, filled)'s polygon: ellipse2Poly's point at k * delta degrees in double with
// the float SinTable, rounded to 16.16 as EllipseEx does.  For r >= 1 pixel no two neighbours coincide, so the
// dedup EllipseEx applies never drops a point.
struct CapPoly {
  int64_t cx, cy, r;
  int delta, n;
  __device__ CapPoly(int64_t cx_, int64_t cy_, int64_t r_) : cx(cx_), cy(cy_), r(r_) {
    const int64_t d = (r + (1 << 15)) >> 16;
    delta = d < 3 ? 90 : d < 10 ? 30 : d < 15 ? 18 : 5;
    n = 360 / delta + 1;
  }
  __device__ static int64_t round16(double v) {
    const int64_t q = __double2ll_rn(__ddiv_rn(v, 65536.0)) << 16;
    return q + __double2ll_rn(__dsub_rn(v, (double)q));
  }
  __device__ void at(int k, int64_t& px, int64_t& py) const {
    const int a = min(k * delta, 360);
    const double x = __dmul_rn((double)r, (double)c_sin[450 - a]), y = __dmul_rn((double)r, (double)c_sin[a]);
    px = round16(__dsub_rn(__dadd_rn((double)cx, __dmul_rn(x, 1.0)), __dmul_rn(y, 0.0)));
    py = round16(__dadd_rn(__dadd_rn((double)cy, __dmul_rn(x, 0.0)), __dmul_rn(y, 1.0)));
  }
};

__device__ inline bool seg_misses(int64_t ax, int64_t ay, int64_t bx, int64_t by, int m, int tx0, int ty0, int tx1,
                                  int ty1) {
  return (max(ax, bx) >> 16) + m < tx0 || (min(ax, bx) >> 16) - m > tx1 || (max(ay, by) >> 16) + m < ty0 ||
         (min(ay, by) >> 16) - m > ty1;
}

// FillConvexPoly(P, black, LINE_AA, XY_SHIFT): LineAA along every edge from the last vertex round, then the opaque
// scanline fill.  The fill's edge walk is OpenCV's, row by row; every thread runs it alike and paints its own rows.
template <class Poly>
__device__ void fill_poly_aa(Px& p, int w, int h, const Poly& P, int tx0, int ty0, int tx1, int ty1) {
  constexpr int S = 16;
  constexpr int64_t ONE = 1 << S, HALF = ONE >> 1;
  const int n = P.n;
  int64_t ax, ay, xmin, xmax, ymin, ymax;
  P.at(n - 1, ax, ay);
  P.at(0, xmin, ymin);
  xmax = xmin;
  ymax = ymin;
  int imin = 0;
  for (int k = 0; k < n; k++) {
    int64_t bx, by;
    P.at(k, bx, by);
    if (by < ymin) { ymin = by; imin = k; }
    ymax = max(ymax, by);
    xmax = max(xmax, bx);
    xmin = min(xmin, bx);
    if (!seg_misses(ax, ay, bx, by, 4, tx0, ty0, tx1, ty1)) line_aa(p, w, h, ax, ay, bx, by);
    ax = bx;
    ay = by;
  }
  xmin = (xmin + HALF) >> S;
  xmax = (xmax + HALF) >> S;
  ymin = (ymin + HALF) >> S;
  ymax = (ymax + HALF) >> S;
  if (n < 3 || xmax < 0 || ymax < 0 || xmin >= w || ymin >= h) return;
  ymax = min(ymax, (int64_t)h - 1);
  if (xmax < tx0 || xmin > tx1 || ymax < ty0 || ymin > ty1) return;
  int edges = n;
  int e_idx[2] = {imin, imin}, e_di[2] = {1, n - 1};
  int64_t e_x[2] = {-ONE, -ONE}, e_dx[2] = {0, 0}, e_ye[2] = {ymin, ymin};
  for (int64_t y = ymin; y <= ymax && y <= ty1; y++) {
    if (y < ymax || y == ymin) {
#pragma unroll
      for (int i = 0; i < 2; i++) {
        if (y < e_ye[i]) continue;
        int idx0 = e_idx[i];
        const int di = e_di[i];
        int idx = idx0 + di;
        if (idx >= n) idx -= n;
        while (edges-- > 0) {
          int64_t xe, ye, xs, ys;
          P.at(idx, xe, ye);
          const int64_t ty = (ye + HALF) >> S;
          if (ty > y) {
            P.at(idx0, xs, ys);
            e_ye[i] = ty;
            e_dx[i] = ((xe - xs) * 2 + (ty - y)) / (2 * (ty - y));
            e_x[i] = xs;
            e_idx[i] = idx;
            break;
          }
          idx0 = idx;
          idx += di;
          if (idx >= n) idx -= n;
        }
      }
    }
    if (edges < 0) break;
    if (y >= ty0 && y >= 0) {
      const int left = e_x[0] > e_x[1] ? 1 : 0;
      const int64_t x1 = max((e_x[left] + ONE - 1) >> S, (int64_t)0), x2 = min(e_x[1 - left] >> S, (int64_t)w - 1);
      if (p.x >= x1 && p.x <= x2) {
#pragma unroll
        for (int k = 0; k < kPix; k++)
          if (p.y[k] == y) { p.v[k][0] = 0; p.v[k][1] = 0; p.v[k][2] = 0; }
      }
    }
    e_x[0] += e_dx[0];
    e_x[1] += e_dx[1];
  }
}

// ThickLine(p0, p1, thickness >= 2, LINE_AA, flags) in black: the quad, then a round cap at p0 (flags & 1) and p1
// (flags & 2)
__device__ void thick_line_aa(Px& p, int w, int h, int64_t x0, int64_t y0, int64_t x1, int64_t y1, int thickness,
                              int flags, int tx0, int ty0, int tx1, int ty1) {
  const double dx = __dmul_rn((double)(x0 - x1), 1.0 / 65536), dy = __dmul_rn((double)(y1 - y0), 1.0 / 65536);
  double r = __dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy));
  const int odd = thickness & 1;
  const int64_t half = (int64_t)thickness << 15;
  if (fabs(r) > 2.220446049250313e-16) {
    r = __ddiv_rn(__dadd_rn((double)half, odd * 65536 * 0.5), __dsqrt_rn(r));
    const int64_t ex = __double2ll_rn(__dmul_rn(dy, r)), ey = __double2ll_rn(__dmul_rn(dx, r));
    QuadPoly q;
    q.x[0] = x0 + ex; q.y[0] = y0 + ey;
    q.x[1] = x0 - ex; q.y[1] = y0 - ey;
    q.x[2] = x1 - ex; q.y[2] = y1 - ey;
    q.x[3] = x1 + ex; q.y[3] = y1 + ey;
    fill_poly_aa(p, w, h, q, tx0, ty0, tx1, ty1);
  }
  if (flags & 1) fill_poly_aa(p, w, h, CapPoly(x0, y0, half), tx0, ty0, tx1, ty1);
  if (flags & 2) fill_poly_aa(p, w, h, CapPoly(x1, y1, half), tx0, ty0, tx1, ty1);
}

struct Blob {
  int n, classes, with_score, codes;
  const int* tl;
  const int* colors;
  const int* names;                                        // [classes, 2]: (offset, length); length -1: no label
  const unsigned char* codes_base;
};

__host__ __device__ inline Blob view_blob(const void* b) {
  const int* w = static_cast<const int*>(b);
  Blob B;
  B.n = w[0];
  B.classes = w[1];
  B.with_score = w[2];
  B.codes = w[3];
  B.tl = w + kHeaderWords;
  B.colors = B.tl + B.n;
  B.names = B.colors + 3 * B.classes;
  B.codes_base = reinterpret_cast<const unsigned char*>(B.names + 2 * B.classes);
  return B;
}

__host__ __device__ inline size_t blob_bytes(int n, int classes, int codes) {
  return ((size_t)4 * (kHeaderWords + n + 5 * (size_t)classes) + (size_t)codes + 15) / 16 * 16;
}

__global__ void __launch_bounds__(kThreads, 1) plot_kernel(uint8_t* data, const float* boxes, const float* scores,
                                                        const int* labels, const int* counts, int slots,
                                                        const void* blob, int* status) {
  const Blob B = view_blob(blob);
  const int img = blockIdx.y;
  const int64_t* desc = reinterpret_cast<const int64_t*>(data) + 4 * img;
  const int h = (int)desc[1], w = (int)desc[2];
  const int64_t pitch = desc[3];
  uint8_t* pix = data + (size_t)B.n * 32 + desc[0];
  const int tiles_x = (w + kTile - 1) / kTile, tiles_y = (h + kTile - 1) / kTile;
  const int tile = blockIdx.x;
  if (tile >= tiles_x * tiles_y) return;
  const int tx0 = (tile % tiles_x) * kTile, ty0 = (tile / tiles_x) * kTile;
  const int tx1 = min(tx0 + kTile, w) - 1, ty1 = min(ty0 + kTile, h) - 1;
  const int tl = B.tl[img];

  __shared__ int spans[kMaxTl / 2 + 2];                   // the corner circle's half width per row offset
  if (threadIdx.x == 0 && tl >= 2) {
    const int radius = (tl + 1) >> 1;
    for (int k = 0; k <= radius; k++) spans[k] = -1;
    int err = 0, dx = radius, dy = 0, plus = 1, minus = (radius << 1) - 1;
    while (dx >= dy) {
      spans[dy] = max(spans[dy], dx);
      spans[dx] = max(spans[dx], dy);
      dy++;
      err += plus;
      plus += 2;
      const int mask = (err <= 0) - 1;
      err -= minus & mask;
      dx += mask;
      minus -= mask & 2;
    }
  }
  __syncthreads();

  Px p;
  p.x = tx0 + (threadIdx.x & (kTile - 1));
#pragma unroll
  for (int k = 0; k < kPix; k++) {
    p.y[k] = ty0 + (threadIdx.x >> 5) + k * (kThreads / kTile);
    p.in[k] = p.x < w && p.y[k] < h;
    const uint8_t* q = pix + p.y[k] * pitch + 3 * p.x;
#pragma unroll
    for (int c = 0; c < 3; c++) p.v[k][c] = p.in[k] ? q[c] : 0;
  }

  const int count = min(max(counts[img], 0), slots);
  int bad = 0, first_bad = -1;
  __shared__ unsigned char text[YB_PLOT_SUFFIX_MAX + 256];
  __shared__ yb_plot_layout L;
  for (int d = 0; d < count; d++) {
    const size_t slot = (size_t)img * slots + d;
    const int label = labels[slot];
    const float* b = boxes + 4 * slot;
    int flag = 0;
    if (label < 0 || label >= B.classes) flag |= YB_PLOT_BAD_LABEL;
    if (!(isfinite(b[0]) && isfinite(b[1]) && isfinite(b[2]) && isfinite(b[3]))) flag |= YB_PLOT_BAD_BOX;
    if (flag) {
      if (!bad) first_bad = d;
      bad |= flag;
      continue;
    }
    int c[4];
#pragma unroll
    for (int k = 0; k < 4; k++) c[k] = (int)fminf(fmaxf(b[k], -kCoordClamp), kCoordClamp);   // int(): truncation
    const int* col = B.colors + 3 * label;
    const int reach = tl + 2;
    if (!(max(c[0], c[2]) + reach < tx0 || min(c[0], c[2]) - reach > tx1 || max(c[1], c[3]) + reach < ty0 ||
          min(c[1], c[3]) - reach > ty1))
      outline(p, c[0], c[1], c[2], c[3], tl, col, spans);
    const int name_off = B.names[2 * label], name_len = B.names[2 * label + 1];
    if (name_len < 0 || (name_len == 0 && !B.with_score)) continue;    // plot_one_box's `if label:`
    // the text lies right of x0 and within one glyph height (32 units) plus a stroke of (x0, y0): tiles it cannot
    // reach skip the layout
    const int pad = 5 + (32 * tl + 2) / 3 + tl;
    if (c[0] - pad > tx1 || c[1] + pad < ty0 || c[1] - 8 * tl - 6 - pad > ty1) continue;
    __syncthreads();                                       // the previous label is read by every thread
    if (threadIdx.x == 0)
      label_layout(B.codes_base + name_off, min(name_len, 255), B.with_score, scores ? scores[slot] : 0.f, tl, c[0],
                   c[1], text, &L);
    __syncthreads();
    if (L.rect_x1 + pad < tx0) continue;
    set_rect(p, c[0], c[1], L.rect_x1, L.rect_y1, col);
    const int tf = L.thickness, m = 4 + (tf + 1) / 2;
    const int64_t hscale = cv_round((double)tl / 3.0 * 65536.0);
    int64_t view_x = (int64_t)L.org_x << 16;
    const int64_t view_y = ((int64_t)L.org_y << 16) - YB_HS_BASE_LINE * hscale;
    for (int t = 0; t < L.length; t++) {
      const char* g = glyph(text[t]);
      view_x -= (g[0] - 'R') * hscale;
      int64_t px0 = 0, py0 = 0;
      int npts = 0;                                        // points so far in this stroke
      for (const char* q = g + 2; *q; ) {
        if (*q == ' ') { npts = 0; q++; continue; }
        const int64_t px1 = (q[0] - 'R') * hscale + view_x, py1 = (q[1] - 'R') * hscale + view_y;
        q += 2;
        // LineAA writes one step past the end point (up to a pixel), and three pixels around the rounded minor
        // coordinate: it stays within 4 pixels of the segment's box; a thick stroke adds its half width
        if (npts && !seg_misses(px0, py0, px1, py1, m, tx0, ty0, tx1, ty1)) {
          if (tf <= 1)
            line_aa(p, w, h, px0, py0, px1, py1);
          else
            thick_line_aa(p, w, h, px0, py0, px1, py1, tf, npts == 1 ? 3 : 2, tx0, ty0, tx1, ty1);
        }
        px0 = px1;
        py0 = py1;
        npts++;
      }
      view_x += (g[1] - 'R') * hscale;
    }
  }

#pragma unroll
  for (int k = 0; k < kPix; k++) {
    if (!p.in[k]) continue;
    uint8_t* q = pix + p.y[k] * pitch + 3 * p.x;
#pragma unroll
    for (int c = 0; c < 3; c++) q[c] = (uint8_t)p.v[k][c];
  }
  if (tile == 0 && threadIdx.x == 0) {
    status[2 * img] = bad;
    status[2 * img + 1] = first_bad;
  }
}

}  // namespace

extern "C" int yb_plot_label_layout(const unsigned char* name, int name_len, int with_score, float score, int tl,
                                    int x0, int y0, unsigned char* text, yb_plot_layout* layout) {
  YB_REQUIRE(name || name_len == 0, "yb_plot_label_layout: null name");
  YB_REQUIRE(text && layout, "yb_plot_label_layout: null output");
  YB_REQUIRE(name_len >= 0 && name_len <= 255, "yb_plot_label_layout: name of %d bytes, 0..255 supported", name_len);
  YB_REQUIRE(tl >= 0 && tl <= kMaxTl, "yb_plot_label_layout: line thickness %d outside 0..%d", tl, kMaxTl);
  label_layout(name, name_len, with_score, score, tl, x0, y0, text, layout);
  return YB_OK;
}

extern "C" int yb_plot_workspace_bytes(int n, int classes, size_t names_bytes, size_t* bytes) {
  YB_REQUIRE(n >= 1 && n <= 65535 && classes >= 1 && bytes, "yb_plot_workspace_bytes: bad arguments");
  *bytes = blob_bytes(n, classes, (int)names_bytes);
  return YB_OK;
}

extern "C" int yb_plot_pack(const int* tl, int n, const int* colors, const unsigned char* names, const int* name_len,
                            int classes, int with_score, void* host_blob, size_t bytes) {
  YB_REQUIRE(tl && colors && name_len && host_blob, "yb_plot_pack: null argument");
  YB_REQUIRE(n >= 1 && n <= 65535 && classes >= 1, "yb_plot_pack: %d images, %d classes", n, classes);
  size_t total = 0;
  for (int c = 0; c < classes; c++) {
    YB_REQUIRE(name_len[c] >= -1 && name_len[c] <= 255, "yb_plot_pack: class %d: label of %d bytes, 0..255 supported",
               c, name_len[c]);
    if (name_len[c] > 0) total += (size_t)name_len[c];
  }
  YB_REQUIRE(total == 0 || names, "yb_plot_pack: null names");
  YB_REQUIRE(bytes >= blob_bytes(n, classes, (int)total), "yb_plot_pack: blob of %zu bytes, %zu needed", bytes,
             blob_bytes(n, classes, (int)total));
  for (int i = 0; i < n; i++) {
    YB_REQUIRE(tl[i] >= 0 && tl[i] <= kMaxTl, "yb_plot_pack: image %d: line thickness %d outside 0..%d", i, tl[i],
               kMaxTl);

  }
  memset(host_blob, 0, bytes);
  int* w = static_cast<int*>(host_blob);
  w[0] = n;
  w[1] = classes;
  w[2] = with_score ? 1 : 0;
  w[3] = (int)total;
  Blob B = view_blob(host_blob);
  memcpy(const_cast<int*>(B.tl), tl, sizeof(int) * n);
  for (int k = 0; k < 3 * classes; k++)                    // cv2 saturates the colour to uchar
    const_cast<int*>(B.colors)[k] = colors[k] < 0 ? 0 : colors[k] > 255 ? 255 : colors[k];
  unsigned char* codes = const_cast<unsigned char*>(B.codes_base);
  int off = 0;
  for (int c = 0; c < classes; c++) {
    const_cast<int*>(B.names)[2 * c] = off;
    const_cast<int*>(B.names)[2 * c + 1] = name_len[c];
    for (int k = 0; k < name_len[c]; k++, off++) codes[off] = (unsigned char)text_code(names[off]);
  }
  return YB_OK;
}

extern "C" int yb_plot_boxes(void* data, int n, int max_pixels_h, int max_pixels_w, const float* boxes,
                             const float* scores, const int* labels, const int* counts, int slots,
                             const void* dev_blob, int* status, void* stream) {
  YB_REQUIRE(data && boxes && labels && counts && dev_blob && status, "yb_plot_boxes: null device pointer");
  YB_REQUIRE(n >= 1 && n <= 65535 && slots >= 0, "yb_plot_boxes: %d images, %d slots", n, slots);
  YB_REQUIRE(max_pixels_h >= 1 && max_pixels_w >= 1, "yb_plot_boxes: empty images");
  const long tiles = (long)((max_pixels_h + kTile - 1) / kTile) * ((max_pixels_w + kTile - 1) / kTile);
  YB_REQUIRE(tiles <= 0x7fffffffL, "yb_plot_boxes: images too large");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  plot_kernel<<<dim3((unsigned)tiles, (unsigned)n), kThreads, 0, st>>>(static_cast<uint8_t*>(data), boxes, scores,
                                                                      labels, counts, slots, dev_blob, status);
  YB_CUDA(cudaGetLastError());
  return YB_OK;
}
