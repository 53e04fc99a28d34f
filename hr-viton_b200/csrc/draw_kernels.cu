// draw_kernels.cu — the ImageDraw shapes of cp_dataset.get_agnostic and get_parse_agnostic.get_im_parse_agnostic rasterised on the
// device, pixel for pixel as Pillow 12.2 draws them in mode 'L' (include/hrviton_sm100_data.h: hrv_agnostic_bits,
// hrv_parse_agnostic).  uint8 / fp64 in, uint8 out, compiled once.
//
// Two launches.  draw_setup_kernel (one block per sample) does the reference's geometry in fp64 from the (25, 2) keypoints and
// turns every shape into a descriptor; its threads then walk each filled ellipse's quarter curve once and store the span of every
// canvas row it covers.  draw_rows_kernel (one block per canvas row of one sample) lets each thread turn one shape into that row's
// spans, then ORs the spans' bits into the row's pixels and writes the row once.
//
// The rules, from Pillow's draw.c and _imaging.c as its output shows them (tests/draw_oracle.py states them in numpy and
// tests/test_draw_cpu.py holds that statement to ImageDraw on random shapes):
//  * Coordinates reach draw.c as C ints: (int) truncation of the double for ellipse, rectangle, line end points and polygon
//    vertices.  x86-64 converts NaN and out-of-range values to INT_MIN; cint() does the same, and int arithmetic wraps (the hip
//    rescaling divides by zero when both hips are missing, and the reference draws those NaN shapes).
//  * hline(x0, y, x1) clips y to [0, h) and x to [0, w); a point is drawn when it lies on the canvas.
//  * Filled ellipse (x0, y0, x1, y1): a = x1 - x0, b = y1 - y0; nothing when a + b < 1.  A walk over the upper-right quarter in
//    doubled coordinates starts at (a, b % 2) and ends at (a % 2, b); each step moves to the candidate nearest the curve
//    b^2 x^2 + a^2 y^2 = a^2 b^2 among (x, y + 2), then (x - 2, y + 2), then (x - 2, y) (a later candidate only when strictly
//    nearer, the x - 2 ones only while x > 1).  With X the first (largest) abscissa on row Y, rows y0 + (b +- Y) / 2 cover columns
//    x0 + (a - X) / 2 .. x0 + (a + X) / 2.
//  * Filled rectangle: rows max(y0, 0) .. min(y1, h), each hline(x0, y, x1).
//  * Wide line (width > 1): dx = x1 - x0, dy = y1 - y0; a zero-length line is the point (x0, y0).  Otherwise with
//    L = hypot(dx, dy), s = (width - 1) / 2, rmax = ROUND_UP(s) / L, rmin = ROUND_DOWN(s) / L (ROUND_UP: half away from zero,
//    ROUND_DOWN: half toward zero) and dxmin = ROUND_DOWN(rmin dy), dxmax = ROUND_DOWN(rmax dy), dymin = ROUND_DOWN(rmin dx),
//    dymax = ROUND_DOWN(rmax dx), the line is the polygon (x0 - dxmin, y0 + dymax), (x1 - dxmin, y1 + dymax),
//    (x1 + dxmax, y1 - dymin), (x0 + dxmax, y0 - dymin).  (Lines of width <= 1 are Bresenham's; neither caller draws one: the
//    narrowest line is get_agnostic's r * 6 with r >= 1.)
//  * Filled polygon: edges between consecutive vertices, plus the closing edge unless the last vertex equals the first.  A
//    horizontal edge is one hline.  The others, with dx = (float)(x1 - x0) / (y1 - y0), are scanned over rows
//    max(ymin, 0) .. min(ymax, h) of the whole polygon (ymin starting from h - 1 and ymax from 0): on row y each edge whose
//    [ymin, ymax] holds y gives x = (y - y0) * dx + x0 in fp32; on the edge's last row it counts twice unless that is the
//    polygon's last row.  An integral x of a sloped edge that an earlier edge with the same sign of dx (covering y) also reaches
//    (after roundf) may move: with off = -1 on the edge's last row and +1 otherwise, and both edges' x on row y + off (the earlier
//    edge covering that row), x moves to roundf(max) + 1 when it lies more than 1 beyond both, or roundf(min) - 1 when more than 1
//    before both; only the first such earlier edge is considered.  The sorted x pair up; each pair fills
//    ROUND_UP(x_a) .. ROUND_DOWN(x_b), both rounded in fp32, when not empty.
//  All fp32 and fp64 arithmetic here is written with _rn intrinsics so that no multiply-add is contracted, except the one fused
//  multiply-add that numpy's 2-vector norm performs (OpenBLAS's ddot on an FMA-capable host: sqrt(fma(y, y, x * x))).
#include <cstdint>

#include "hrv_host.h"
#include "../../include/hrviton_sm100_data.h"

namespace hrv_draw {
using hrv_host::set_error;

constexpr int kMaxShapes = 32;
constexpr int kMaxEllipses = 16;
constexpr int kMaxSpans = 8;  // per shape and row: 4 scanned pairs of a 4-edge polygon + 4 horizontal edges
constexpr int kRowThreads = 128;
constexpr int INT_MIN_ = (int)0x80000000;

enum Kind { NONE = 0, ELLIPSE = 1, POLY = 2, RECT = 3, POINT = 4 };

struct Edge {
  int xmin, xmax, ymin, ymax, x0, y0;
  float dx;
};

struct Shape {
  int kind, bit, n_edges, slot;  // slot: the ellipse's rows in the table
  int x0, y0, x1, y1;            // ellipse / rectangle box, point
  Edge e[4];
};

struct Workspace {  // per sample
  int n_shapes;
  int pad[3];
  Shape shape[kMaxShapes];
};

__device__ __forceinline__ int iadd(int a, int b) { return (int)((unsigned)a + (unsigned)b); }
__device__ __forceinline__ int isub(int a, int b) { return (int)((unsigned)a - (unsigned)b); }

// (int)v on x86-64: truncation; NaN and values outside int32 give INT_MIN
__device__ __forceinline__ int cint(double v) { return (v > -2147483649.0 && v < 2147483648.0) ? (int)v : INT_MIN_; }
__device__ __forceinline__ int round_up(double f) { return cint(f >= 0.0 ? floor(__dadd_rn(f, 0.5)) : -floor(__dadd_rn(fabs(f), 0.5))); }
__device__ __forceinline__ int round_down(double f) { return cint(f >= 0.0 ? ceil(__dadd_rn(f, -0.5)) : -ceil(__dadd_rn(fabs(f), -0.5))); }
__device__ __forceinline__ int round_up_f(float f) {
  return cint(f >= 0.f ? floor((double)__fadd_rn(f, 0.5f)) : -floor((double)__fadd_rn(fabsf(f), 0.5f)));
}
__device__ __forceinline__ int round_down_f(float f) {
  return cint(f >= 0.f ? ceil((double)__fadd_rn(f, -0.5f)) : -ceil((double)__fadd_rn(fabsf(f), -0.5f)));
}

__device__ Edge make_edge(int x0, int y0, int x1, int y1) {
  Edge e;
  e.xmin = min(x0, x1), e.xmax = max(x0, x1), e.ymin = min(y0, y1), e.ymax = max(y0, y1), e.x0 = x0, e.y0 = y0;
  e.dx = y0 == y1 ? 0.f : __fdiv_rn((float)isub(x1, x0), (float)isub(y1, y0));
  return e;
}

__device__ __forceinline__ float edge_x(const Edge& e, int y) { return __fadd_rn(__fmul_rn((float)isub(y, e.y0), e.dx), (float)e.x0); }

// ------------------------------------------------------------------------------------------------ shape builders (setup thread)
struct Builder {
  Shape* s;
  int n, n_ellipses;

  __device__ void ellipse(double x0, double y0, double x1, double y1, int bit) {
    Shape& t = s[n++];
    t.kind = ELLIPSE, t.bit = bit, t.slot = n_ellipses++;
    t.x0 = cint(x0), t.y0 = cint(y0), t.x1 = cint(x1), t.y1 = cint(y1);
  }
  __device__ void rectangle(double x0, double y0, double x1, double y1, int bit) {
    Shape& t = s[n++];
    t.kind = RECT, t.bit = bit;
    t.x0 = cint(x0), t.y0 = cint(y0), t.x1 = cint(x1), t.y1 = cint(y1);
  }
  __device__ void polygon(const double (*p)[2], int count, int bit) {  // count <= 4
    Shape& t = s[n++];
    t.kind = POLY, t.bit = bit, t.n_edges = 0;
    int v[4][2];
    for (int i = 0; i < count; ++i) v[i][0] = cint(p[i][0]), v[i][1] = cint(p[i][1]);
    for (int i = 0; i + 1 < count; ++i) t.e[t.n_edges++] = make_edge(v[i][0], v[i][1], v[i + 1][0], v[i + 1][1]);
    if (v[count - 1][0] != v[0][0] || v[count - 1][1] != v[0][1])
      t.e[t.n_edges++] = make_edge(v[count - 1][0], v[count - 1][1], v[0][0], v[0][1]);
  }
  __device__ void line(const double* p, const double* q, int width, int bit) {  // width > 1
    const int x0 = cint(p[0]), y0 = cint(p[1]), x1 = cint(q[0]), y1 = cint(q[1]);
    const int dx = isub(x1, x0), dy = isub(y1, y0);
    Shape& t = s[n++];
    t.bit = bit;
    if (dx == 0 && dy == 0) {
      t.kind = POINT, t.x0 = x0, t.y0 = y0;
      return;
    }
    const double big = __dsqrt_rn(__dadd_rn(__dmul_rn((double)dx, (double)dx), __dmul_rn((double)dy, (double)dy)));  // hypot
    const double small = (width - 1) / 2.0;
    const double rmax = __ddiv_rn((double)round_up(small), big), rmin = __ddiv_rn((double)round_down(small), big);
    const int dxmin = round_down(__dmul_rn(rmin, (double)dy)), dxmax = round_down(__dmul_rn(rmax, (double)dy));
    const int dymin = round_down(__dmul_rn(rmin, (double)dx)), dymax = round_down(__dmul_rn(rmax, (double)dx));
    const int v[4][2] = {{isub(x0, dxmin), iadd(y0, dymax)}, {isub(x1, dxmin), iadd(y1, dymax)},
                         {iadd(x1, dxmax), isub(y1, dymin)}, {iadd(x0, dxmax), isub(y0, dymin)}};
    t.kind = POLY, t.n_edges = 4;
    for (int i = 0; i < 4; ++i) t.e[i] = make_edge(v[i][0], v[i][1], v[(i + 1) & 3][0], v[(i + 1) & 3][1]);
  }
};

__device__ __forceinline__ bool absent(const double (*p)[2], int i) { return p[i][0] == 0.0 && p[i][1] == 0.0; }

// numpy's np.linalg.norm(a - b) of two points
__device__ __forceinline__ double norm2(const double* a, const double* b) {
  const double dx = __dadd_rn(a[0], -b[0]), dy = __dadd_rn(a[1], -b[1]);
  return __dsqrt_rn(__fma_rn(dy, dy, __dmul_rn(dx, dx)));
}

// cp_dataset.get_agnostic: bit 0 the grey shapes, bits 1 / 2 the label-14 / label-15 arm masks
__device__ void agnostic_shapes(double (*p)[2], Builder& b) {
  const double shoulders = norm2(p[5], p[2]), hips = norm2(p[12], p[9]);
  double mid[2];
  for (int c = 0; c < 2; ++c) mid[c] = __dadd_rn(p[9][c], p[12][c]) / 2.0;
  for (int c = 0; c < 2; ++c) {
    p[9][c] = __dadd_rn(mid[c], __dmul_rn(__ddiv_rn(__dadd_rn(p[9][c], -mid[c]), hips), shoulders));
    p[12][c] = __dadd_rn(mid[c], __dmul_rn(__ddiv_rn(__dadd_rn(p[12][c], -mid[c]), hips), shoulders));
  }
  const int r = (int)(shoulders / 16.0) + 1;
  auto box = [&](int i, int rx, int ry, int bit) {
    b.ellipse(__dadd_rn(p[i][0], -(double)(r * rx)), __dadd_rn(p[i][1], -(double)(r * ry)), __dadd_rn(p[i][0], (double)(r * rx)),
              __dadd_rn(p[i][1], (double)(r * ry)), bit);
  };
  box(9, 3, 6, 1);  // torso
  box(12, 3, 6, 1);
  b.line(p[2], p[9], r * 6, 1);
  b.line(p[5], p[12], r * 6, 1);
  b.line(p[9], p[12], r * 12, 1);
  const double quad[4][2] = {{p[2][0], p[2][1]}, {p[5][0], p[5][1]}, {p[12][0], p[12][1]}, {p[9][0], p[9][1]}};
  b.polygon(quad, 4, 1);
  b.rectangle(__dadd_rn(p[1][0], -(double)(r * 5)), __dadd_rn(p[1][1], -(double)(r * 9)), __dadd_rn(p[1][0], (double)(r * 5)), p[1][1], 1);
  b.line(p[2], p[5], r * 12, 1);  // arms
  box(2, 5, 6, 1);
  box(5, 5, 6, 1);
  for (int i : {3, 4, 6, 7}) {
    if (absent(p, i - 1) || absent(p, i)) continue;
    b.line(p[i - 1], p[i], r * 10, 1);
    box(i, 5, 5, 1);
  }
  const int arms[2][3] = {{5, 6, 7}, {2, 3, 4}};
  for (int a = 0; a < 2; ++a) {
    const int* j = arms[a];
    const int bit = 2 << a;
    box(j[0], 5, 6, bit);
    int last = j[0];
    for (int k = 1; k < 3; ++k) {
      const int i = j[k];
      if (absent(p, i - 1) || absent(p, i)) continue;
      b.line(p[i - 1], p[i], r * 10, bit);
      last = i;
      if (k != 2) box(i, 5, 5, bit);
    }
    box(last, 4, 4, bit);
  }
}

// get_parse_agnostic.get_im_parse_agnostic: bits 1 / 2 the label-14 / label-15 arm masks (r = 10)
__device__ void parse_shapes(const double (*p)[2], Builder& b) {
  const int ids[2][4] = {{2, 5, 6, 7}, {5, 2, 3, 4}};
  for (int a = 0; a < 2; ++a) {
    int prev = ids[a][0];
    for (int k = 1; k < 4; ++k) {
      const int i = ids[a][k];
      if (absent(p, prev) || absent(p, i)) continue;
      b.line(p[prev], p[i], 100, 2 << a);
      const double radius = k == 3 ? 40.0 : 150.0;
      b.ellipse(__dadd_rn(p[i][0], -radius), __dadd_rn(p[i][1], -radius), __dadd_rn(p[i][0], radius), __dadd_rn(p[i][1], radius), 2 << a);
      prev = i;
    }
  }
}

// One block per sample: thread 0 builds the shapes, then every ellipse's rows are cleared and walked (one thread per ellipse).
template <bool PARSE>
__global__ void __launch_bounds__(64) draw_setup_kernel(const double* __restrict__ keypoints, int h, Workspace* __restrict__ ws,
                                                        short2* __restrict__ rows) {
  __shared__ Shape shapes[kMaxShapes];
  __shared__ int counts[2];
  const int sample = blockIdx.x;
  if (threadIdx.x == 0) {
    double p[25][2];
    for (int i = 0; i < 25; ++i) p[i][0] = keypoints[(sample * 25 + i) * 2], p[i][1] = keypoints[(sample * 25 + i) * 2 + 1];
    Builder b{shapes, 0, 0};
    if (PARSE)
      parse_shapes(p, b);
    else
      agnostic_shapes(p, b);
    counts[0] = b.n, counts[1] = b.n_ellipses;
  }
  __syncthreads();
  const int n_shapes = counts[0];
  Workspace& w = ws[sample];
  if (threadIdx.x == 0) w.n_shapes = n_shapes;
  for (int i = threadIdx.x; i < n_shapes * (int)(sizeof(Shape) / 4); i += blockDim.x)
    reinterpret_cast<int*>(w.shape)[i] = reinterpret_cast<const int*>(shapes)[i];
  short2* table = rows + (long long)sample * kMaxEllipses * h;
  for (int i = threadIdx.x; i < counts[1] * h; i += blockDim.x) table[i] = make_short2(1, 0);  // empty
  __syncthreads();
  for (int s = threadIdx.x; s < n_shapes; s += blockDim.x) {
    const Shape& t = shapes[s];
    if (t.kind != ELLIPSE) continue;
    const long long a = (long long)t.x1 - t.x0, bb = (long long)t.y1 - t.y0;
    const int x0 = t.x0, y0 = t.y0;
    if (a < 0 || bb < 0 || a + bb < 1 || a > 65535 || bb > 65535) continue;  // larger boxes need keypoints the Python layer refuses
    short2* out = table + (long long)t.slot * h;
    const long long a2 = a * a, b2 = bb * bb, a2b2 = a2 * b2;
    auto delta = [&](long long x, long long y) { return llabs(a2 * y * y + b2 * x * x - a2b2); };
    long long cx = a, cy = bb % 2, prev_y = -1;
    const long long ex = a % 2, ey = bb;
    while (true) {
      if (cy != prev_y) {
        prev_y = cy;
        const int xl = iadd(x0, (int)((a - cx) / 2)), xr = iadd(x0, (int)((a + cx) / 2));
        const int ylo = iadd(y0, (int)((bb - cy) / 2)), yhi = iadd(y0, (int)((bb + cy) / 2));
        const short2 span = make_short2((short)min(max(xl, 0), 32767), (short)max(min(xr, 32767), -1));
        if (ylo >= 0 && ylo < h) out[ylo] = span;
        if (yhi >= 0 && yhi < h) out[yhi] = span;
        if (ylo < 0 && yhi >= h) break;  // every later row lies off the canvas
      }
      if (cx == ex && cy == ey) break;
      long long nx = cx, ny = cy + 2, nd = delta(nx, ny);
      if (nx > 1) {
        long long d = delta(cx - 2, cy + 2);
        if (nd > d) nx = cx - 2, ny = cy + 2, nd = d;
        d = delta(cx - 2, cy);
        if (nd > d) nx = cx - 2, ny = cy;
      }
      cx = nx, cy = ny;
    }
  }
}

struct Span {
  int x0, x1, bit;
};

// The spans of polygon `t` on row y (before x clipping), appended at `out`; returns the count.
__device__ int polygon_row(const Shape& t, int y, int h, Span* out) {
  int n = 0, ymin = h - 1, ymax = 0;
  for (int i = 0; i < t.n_edges; ++i) {
    const Edge& e = t.e[i];
    ymin = min(ymin, e.ymin), ymax = max(ymax, e.ymax);
    if (e.ymin == e.ymax && e.ymin == y) out[n++] = {e.xmin, e.xmax, t.bit};
  }
  ymin = max(ymin, 0), ymax = min(ymax, h);
  if (y < ymin || y > ymax) return n;
  float xx[8];
  int j = 0;
  const Edge* table[4];
  int m = 0;
  for (int i = 0; i < t.n_edges; ++i)
    if (t.e[i].ymin != t.e[i].ymax) table[m++] = &t.e[i];
  for (int i = 0; i < m; ++i) {
    const Edge& cur = *table[i];
    if (y < cur.ymin || y > cur.ymax) continue;
    xx[j++] = edge_x(cur, y);
    if (y == cur.ymax && y < ymax) {
      xx[j] = xx[j - 1];
      ++j;
    } else if (cur.dx != 0.f && roundf(xx[j - 1]) == xx[j - 1]) {
      for (int k = 0; k < i; ++k) {
        const Edge& o = *table[k];
        if ((cur.dx > 0.f && o.dx <= 0.f) || (cur.dx < 0.f && o.dx >= 0.f) || y < o.ymin || y > o.ymax) continue;
        if (roundf(xx[j - 1]) != roundf(edge_x(o, y))) continue;
        const int yo = iadd(y, y == cur.ymax ? -1 : 1);
        const float adj = edge_x(cur, yo);
        if (yo < o.ymin || yo > o.ymax) continue;
        const float adj_o = edge_x(o, yo);
        const float v = xx[j - 1];
        if (v > __fadd_rn(adj, 1.f) && v > __fadd_rn(adj_o, 1.f))
          xx[j - 1] = __fadd_rn(roundf(fmaxf(adj, adj_o)), 1.f);
        else if (v < __fadd_rn(adj, -1.f) && v < __fadd_rn(adj_o, -1.f))
          xx[j - 1] = __fadd_rn(roundf(fminf(adj, adj_o)), -1.f);
        break;
      }
    }
  }
  for (int a = 1; a < j; ++a)  // insertion sort, ascending
    for (int b = a; b > 0 && xx[b - 1] > xx[b]; --b) {
      const float tmp = xx[b];
      xx[b] = xx[b - 1], xx[b - 1] = tmp;
    }
  for (int k = 1; k < j; k += 2) {
    const int x0 = round_up_f(xx[k - 1]), x1 = round_down_f(xx[k]);
    if (x1 >= x0) out[n++] = {x0, x1, t.bit};
  }
  return n;
}

// One block per (row, sample).  PARSE: out = the label row with get_im_parse_agnostic's pastes applied; else the bit row.
template <bool PARSE>
__global__ void __launch_bounds__(kRowThreads) draw_rows_kernel(const Workspace* __restrict__ ws, const short2* __restrict__ rows,
                                                                const unsigned char* __restrict__ labels, int h, int w,
                                                                unsigned char* __restrict__ out) {
  __shared__ Span spans[kMaxShapes * kMaxSpans];
  __shared__ int n_spans;
  const int y = blockIdx.x, sample = blockIdx.y;
  const Workspace& wsp = ws[sample];
  if (threadIdx.x == 0) n_spans = 0;
  __syncthreads();
  const int n_shapes = wsp.n_shapes;
  for (int s = threadIdx.x; s < n_shapes; s += blockDim.x) {
    const Shape& t = wsp.shape[s];
    Span local[kMaxSpans];
    int n = 0;
    if (t.kind == ELLIPSE) {
      const short2 r = rows[((long long)sample * kMaxEllipses + t.slot) * h + y];
      if (r.x <= r.y) local[n++] = {r.x, r.y, t.bit};
    } else if (t.kind == RECT) {
      if (y >= t.y0 && y <= t.y1) local[n++] = {t.x0, t.x1, t.bit};
    } else if (t.kind == POINT) {
      if (y == t.y0) local[n++] = {t.x0, t.x0, t.bit};
    } else if (t.kind == POLY) {
      n = polygon_row(t, y, h, local);
    }
    int at = n ? atomicAdd(&n_spans, n) : 0;
    for (int i = 0; i < n; ++i) spans[at + i] = local[i];
  }
  __syncthreads();
  const int ns = n_spans;
  const long long row = ((long long)sample * h + y) * w;
  for (int x = threadIdx.x; x < w; x += blockDim.x) {
    int bits = 0;
    for (int i = 0; i < ns; ++i)
      if (x >= spans[i].x0 && x <= spans[i].x1) bits |= spans[i].bit;
    if (PARSE) {
      const int l = labels[row + x];
      const bool clear = ((bits & 2) && l == 14) || ((bits & 4) && l == 15) || l == 5 || l == 6 || l == 7 || l == 10;
      out[row + x] = clear ? 0 : (unsigned char)l;
    } else {
      out[row + x] = (unsigned char)bits;
    }
  }
}

size_t workspace_bytes(int n, int h) {
  return (size_t)n * sizeof(Workspace) + (size_t)n * kMaxEllipses * h * sizeof(short2);
}

template <bool PARSE>
int launch(const double* keypoints, const uint8_t* labels, int n, int h, int w, uint8_t* out, void* workspace, size_t ws_bytes,
           cudaStream_t st, const char* what) {
  if (!keypoints || !out || !workspace || (PARSE && !labels) || n < 0 || h <= 0 || w <= 0 || h > 32767 || w > 32767)
    return set_error(HRV_EINVAL, "%s: bad arguments (n %d, h %d, w %d)", what, n, h, w);
  if (ws_bytes < workspace_bytes(n, h))
    return set_error(HRV_EINVAL, "%s: workspace of %zu bytes, need %zu", what, ws_bytes, workspace_bytes(n, h));
  if (n == 0) return HRV_OK;
  Workspace* wsp = static_cast<Workspace*>(workspace);
  short2* rows = reinterpret_cast<short2*>(wsp + n);
  draw_setup_kernel<PARSE><<<n, 64, 0, st>>>(keypoints, h, wsp, rows);
  draw_rows_kernel<PARSE><<<dim3(h, n), kRowThreads, 0, st>>>(wsp, rows, labels, h, w, out);
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? HRV_OK : set_error(HRV_ECUDA, "%s: %s", what, cudaGetErrorString(e));
}
}  // namespace hrv_draw

extern "C" {
size_t hrv_draw_workspace_bytes(int32_t n, int32_t h) { return hrv_draw::workspace_bytes(n, h); }

int hrv_agnostic_bits(const double* keypoints, int32_t n, int32_t h, int32_t w, uint8_t* bits, void* workspace, size_t workspace_bytes,
                      hrv_stream stream) {
  return hrv_draw::launch<false>(keypoints, nullptr, n, h, w, bits, workspace, workspace_bytes, (cudaStream_t)stream, "agnostic_bits");
}

int hrv_parse_agnostic(const double* keypoints, const uint8_t* labels, int32_t n, int32_t h, int32_t w, uint8_t* out, void* workspace,
                       size_t workspace_bytes, hrv_stream stream) {
  return hrv_draw::launch<true>(keypoints, labels, n, h, w, out, workspace, workspace_bytes, (cudaStream_t)stream, "parse_agnostic");
}
}
