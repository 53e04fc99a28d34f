"""numpy restatement of the ImageDraw primitives that cp_dataset.get_agnostic and get_parse_agnostic.get_im_parse_agnostic draw (Pillow
12.2, mode 'L', one ink, no antialiasing), written as the scanline rules csrc/draw_kernels.cu runs: every shape is a set of
horizontal spans (hline), clipped to the canvas.  C semantics are kept where they decide a pixel: float -> int conversion truncates
and gives INT_MIN for NaN or out-of-range values (x86 cvttsd2si), int arithmetic wraps at 32 bits, polygon scanline intersections
are fp32 without fused multiply-add."""
import math

import numpy as np

INT_MIN = -(1 << 31)
F32 = np.float32


def wrap(v):
    """v as a C int32 (two's-complement wrap)."""
    return ((int(v) + (1 << 31)) & 0xFFFFFFFF) - (1 << 31)


def cint(v):
    """(int)v for a double v as x86-64 does it: truncation, INT_MIN for NaN and out-of-range values."""
    v = float(v)
    if math.isnan(v) or not (-2147483649.0 < v < 2147483648.0):
        return INT_MIN
    return int(v)


def round_up(f):
    """draw.c's ROUND_UP for a double: half away from zero."""
    f = float(f)
    return cint(math.floor(f + 0.5) if f >= 0.0 else -math.floor(abs(f) + 0.5))


def round_down(f):
    """draw.c's ROUND_DOWN for a double: half toward zero."""
    f = float(f)
    return cint(math.ceil(f - 0.5) if f >= 0.0 else -math.ceil(abs(f) - 0.5))


def round_up_f32(f):
    """ROUND_UP of a float: the + 0.5F is an fp32 add."""
    f = F32(f)
    return cint(math.floor(F32(f + F32(0.5))) if f >= 0 else -math.floor(F32(abs(f) + F32(0.5))))


def round_down_f32(f):
    f = F32(f)
    return cint(math.ceil(F32(f - F32(0.5))) if f >= 0 else -math.ceil(F32(abs(f) - F32(0.5))))


class Canvas:
    """A w x h boolean mask with draw.c's clipped hline and point."""

    def __init__(self, w, h):
        self.w, self.h = w, h
        self.m = np.zeros((h, w), bool)

    def hline(self, x0, y, x1):
        if 0 <= y < self.h:
            x0, x1 = max(x0, 0), min(x1, self.w - 1)
            if x0 <= x1:
                self.m[y, x0:x1 + 1] = True

    def point(self, x, y):
        if 0 <= x < self.w and 0 <= y < self.h:
            self.m[y, x] = True

    # ---------------------------------------------------------------------------------------------------- ellipse (filled)
    def ellipse(self, xy):
        """ImageDraw.ellipse(xy, fill): the corners truncate to int; the quarter-ellipse walk below runs in doubled coordinates
        and row (b +- Y) / 2 covers columns (a - X) / 2 .. (a + X) / 2, X the largest abscissa the walk visits on that row."""
        x0, y0, x1, y1 = (float(v) for v in xy)
        if x1 < x0 or y1 < y0:
            raise ValueError("ellipse box out of order")
        x0, y0, x1, y1 = cint(x0), cint(y0), cint(x1), cint(y1)
        a, b = wrap(x1 - x0), wrap(y1 - y0)
        for X, Y in ellipse_rows(a, b):
            for yy in {Y, -Y}:
                self.hline(wrap(x0 + (a - X) // 2), wrap(y0 + (b + yy) // 2), wrap(x0 + (a + X) // 2))

    # ---------------------------------------------------------------------------------------------------- rectangle (filled)
    def rectangle(self, xy):
        x0, y0, x1, y1 = (float(v) for v in xy)
        if x1 < x0 or y1 < y0:
            raise ValueError("rectangle box out of order")
        x0, y0, x1, y1 = cint(x0), cint(y0), cint(x1), cint(y1)
        for y in range(max(y0, 0), min(y1, self.h - 1) + 1):
            self.hline(x0, y, x1)

    # ---------------------------------------------------------------------------------------------------- polygon (filled)
    def polygon(self, pts):
        """ImageDraw.polygon(pts, fill): vertices truncate to int, then draw.c's polygon scan over the closed edge list."""
        v = [(cint(x), cint(y)) for x, y in pts]
        edges = [(v[i], v[i + 1]) for i in range(len(v) - 1)]
        if v[-1] != v[0]:
            edges.append((v[-1], v[0]))
        self.scan([make_edge(*p, *q) for p, q in edges])

    def scan(self, edges):
        for y, x0, x1 in polygon_spans(edges, self.h):
            self.hline(x0, y, x1)

    # ---------------------------------------------------------------------------------------------------- line
    def line(self, p, q, width):
        """ImageDraw.line([p, q], fill, width): the end points truncate to int.  width <= 1 is Bresenham's line plus its end point;
        a wider line is the 4-vertex polygon draw.c's ImagingDrawWideLine builds; a zero-length wide line is one point."""
        x0, y0, x1, y1 = cint(p[0]), cint(p[1]), cint(q[0]), cint(q[1])
        if width <= 1:
            for x, y in bresenham(x0, y0, x1, y1):
                self.point(x, y)
            self.point(x1, y1)
            return
        quad = wide_line_quad(x0, y0, x1, y1, width)
        if quad is None:
            self.point(x0, y0)
            return
        self.scan([make_edge(*quad[i], *quad[(i + 1) % 4]) for i in range(4)])


def ellipse_rows(a, b):
    """(X, Y) per row of the upper-right quarter of an a x b filled ellipse, in doubled coordinates: the walk starts at (a, b % 2)
    and ends at (a % 2, b); each step takes the nearest of (x, y + 2), (x - 2, y + 2), (x - 2, y) to the curve
    b^2 x^2 + a^2 y^2 = a^2 b^2 (the later candidate only on a strictly smaller |deviation|; x - 2 only while x > 1).  A filled
    ellipse of width a + b draws nothing if a + b < 1, i.e. a single pixel needs a one-pixel box."""
    if a < 0 or b < 0 or a + b < 1:
        return []
    a2, b2 = a * a, b * b
    a2b2 = a2 * b2

    def delta(x, y):
        return abs(a2 * y * y + b2 * x * x - a2b2)
    cx, cy, ex, ey = a, b % 2, a % 2, b
    rows = []
    while True:
        if not rows or rows[-1][1] != cy:
            rows.append((cx, cy))
        if cx == ex and cy == ey:
            break
        nx, ny = cx, cy + 2
        nd = delta(nx, ny)
        if nx > 1:
            d = delta(cx - 2, cy + 2)
            if nd > d:
                nx, ny, nd = cx - 2, cy + 2, d
            d = delta(cx - 2, cy)
            if nd > d:
                nx, ny = cx - 2, cy
        cx, cy = nx, ny
    return rows


def bresenham(x0, y0, x1, y1):
    """The points draw.c's line8 visits (the end point excluded)."""
    dx, xs = (x1 - x0, 1) if x1 >= x0 else (x0 - x1, -1)
    dy, ys = (y1 - y0, 1) if y1 >= y0 else (y0 - y1, -1)
    out = []
    if dx == 0:
        for _ in range(dy):
            out.append((x0, y0))
            y0 += ys
    elif dy == 0:
        for _ in range(dx):
            out.append((x0, y0))
            x0 += xs
    elif dx > dy:
        n, dy2, dx2 = dx, dy + dy, dx + dx
        e = dy2 - dx
        for _ in range(n):
            out.append((x0, y0))
            if e >= 0:
                y0 += ys
                e -= dx2
            e += dy2
            x0 += xs
    else:
        n, dx2, dy2 = dy, dx + dx, dy + dy
        e = dx2 - dy
        for _ in range(n):
            out.append((x0, y0))
            if e >= 0:
                x0 += xs
                e -= dy2
            e += dx2
            y0 += ys
    return out


def wide_line_quad(x0, y0, x1, y1, width):
    """The corners of ImagingDrawWideLine's polygon, or None for a zero-length segment."""
    dx, dy = wrap(x1 - x0), wrap(y1 - y0)
    if dx == 0 and dy == 0:
        return None
    big = math.hypot(dx, dy)
    small = (width - 1) / 2.0
    ratio_max = round_up(small) / big
    ratio_min = round_down(small) / big
    dxmin, dxmax = round_down(ratio_min * dy), round_down(ratio_max * dy)
    dymin, dymax = round_down(ratio_min * dx), round_down(ratio_max * dx)
    return [(wrap(x0 - dxmin), wrap(y0 + dymax)), (wrap(x1 - dxmin), wrap(y1 + dymax)),
            (wrap(x1 + dxmax), wrap(y1 - dymin)), (wrap(x0 + dxmax), wrap(y0 - dymin))]


def make_edge(x0, y0, x1, y1):
    """draw.c's add_edge: (xmin, xmax, ymin, ymax, x0, y0, dx) with dx = (float)(x1 - x0) / (y1 - y0) in fp32."""
    dx = F32(0) if y0 == y1 else F32(F32(wrap(x1 - x0)) / F32(wrap(y1 - y0)))
    return (min(x0, x1), max(x0, x1), min(y0, y1), max(y0, y1), x0, y0, dx)


def _at(e, y):
    """(y - y0) * dx + x0 in fp32, as the scan computes an edge's intersection with row y."""
    return F32(F32(F32(wrap(y - e[5])) * e[6]) + F32(e[4]))


def polygon_spans(edges, height):
    """(y, x_start, x_end) of every span draw.c's polygon_generic fills, unclipped in x, for rows clipped to [0, height]."""
    spans = []
    table = []
    ymin, ymax = height - 1, 0
    for e in edges:
        ymin, ymax = min(ymin, e[2]), max(ymax, e[3])
        if e[2] == e[3]:
            spans.append((e[2], e[0], e[1]))  # horizontal edge
            continue
        table.append(e)
    ymin, ymax = max(ymin, 0), min(ymax, height)
    for y in range(ymin, ymax + 1):
        xx = []
        for i, cur in enumerate(table):
            if not (cur[2] <= y <= cur[3]):
                continue
            xx.append(_at(cur, y))
            if y == cur[3] and y < ymax:
                xx.append(xx[-1])  # an edge's last row counts twice except on the polygon's last row
            elif cur[6] != 0 and F32(np.round(xx[-1])) == xx[-1]:
                _corner(table, i, cur, y, xx)
        xx.sort()
        for k in range(1, len(xx), 2):
            x0, x1 = round_up_f32(xx[k - 1]), round_down_f32(xx[k])
            if x1 >= x0:
                spans.append((y, x0, x1))
    return spans


def _roundf(v):
    """C roundf: half away from zero."""
    v = F32(v)
    return F32(math.floor(abs(v) + 0.5) * (1 if v >= 0 else -1)) if abs(v) < 2 ** 23 else v


def _corner(table, i, cur, y, xx):
    """polygon_generic's 'connect discontiguous corners' rule: an integral intersection that an earlier edge of the same slope
    direction shares moves one pixel past both edges' intersections with the next (or, on the edge's last row, previous) row when
    it lies more than a pixel beyond both."""
    for k in range(i):
        other = table[k]
        if (cur[6] > 0 and other[6] <= 0) or (cur[6] < 0 and other[6] >= 0) or not (other[2] <= y <= other[3]):
            continue
        if _roundf(xx[-1]) != _roundf(_at(other, y)):
            continue
        off = -1 if y == cur[3] else 1
        adj = _at(cur, y + off)
        if not (other[2] <= y + off <= other[3]):
            continue
        adj_o = _at(other, y + off)
        if xx[-1] > F32(adj + F32(1)) and xx[-1] > F32(adj_o + F32(1)):
            xx[-1] = F32(_roundf(max(adj, adj_o)) + F32(1))
        elif xx[-1] < F32(adj - F32(1)) and xx[-1] < F32(adj_o - F32(1)):
            xx[-1] = F32(_roundf(min(adj, adj_o)) - F32(1))
        break


# ---------------------------------------------------------------------------------------------------- the two callers, restated
def _norm(a, b):
    """np.linalg.norm(a - b) of two points as numpy computes it on an FMA host: sqrt(fma(y, y, x * x))."""
    from fractions import Fraction
    x, y = float(a[0] - b[0]), float(a[1] - b[1])
    return math.sqrt(float(Fraction(y) * Fraction(y) + Fraction(x * x)))


def agnostic_bits(pose, size=(768, 1024)):
    """data.agnostic_bits through the restated primitives."""
    p = np.array(pose, dtype=np.float64)[:25]
    shoulders, hips = np.linalg.norm(p[5] - p[2]), np.linalg.norm(p[12] - p[9])
    mid = (p[9] + p[12]) / 2
    with np.errstate(all="ignore"):
        p[9] = mid + (p[9] - mid) / hips * shoulders
        p[12] = mid + (p[12] - mid) / hips * shoulders
    r = int(shoulders / 16) + 1

    def box(i, rx, ry):
        return (p[i][0] - r * rx, p[i][1] - r * ry, p[i][0] + r * rx, p[i][1] + r * ry)

    def absent(i):
        return p[i, 0] == 0.0 and p[i, 1] == 0.0
    c = Canvas(*size)
    for i in (9, 12):
        c.ellipse(box(i, 3, 6))
    c.line(p[2], p[9], r * 6)
    c.line(p[5], p[12], r * 6)
    c.line(p[9], p[12], r * 12)
    c.polygon([p[2], p[5], p[12], p[9]])
    x, y = p[1]
    c.rectangle((x - r * 5, y - r * 9, x + r * 5, y))
    c.line(p[2], p[5], r * 12)
    for i in (2, 5):
        c.ellipse(box(i, 5, 6))
    for i in (3, 4, 6, 7):
        if not (absent(i - 1) or absent(i)):
            c.line(p[i - 1], p[i], r * 10)
            c.ellipse(box(i, 5, 5))
    bits = c.m.astype(np.uint8)
    for bit, joints in ((1, (5, 6, 7)), (2, (2, 3, 4))):
        a = Canvas(768, 1024)
        a.ellipse(box(joints[0], 5, 6))
        last = joints[0]
        for i in joints[1:]:
            if absent(i - 1) or absent(i):
                continue
            a.line(p[i - 1], p[i], r * 10)
            last = i
            if i != joints[-1]:
                a.ellipse(box(i, 5, 5))
        a.ellipse(box(last, 4, 4))
        bits |= a.m.astype(np.uint8) << bit
    return bits


def parse_agnostic(labels, pose):
    """get_im_parse_agnostic(labels, pose, w, h) through the restated primitives: labels (h, w) uint8 -> (h, w) uint8."""
    p = np.asarray(pose, dtype=np.float64)
    h, w = labels.shape
    clear = np.isin(labels, (5, 6, 7, 10))
    for label, ids in ((14, (2, 5, 6, 7)), (15, (5, 2, 3, 4))):
        c = Canvas(w, h)
        prev = ids[0]
        for i in ids[1:]:
            if (p[prev, 0] == 0.0 and p[prev, 1] == 0.0) or (p[i, 0] == 0.0 and p[i, 1] == 0.0):
                continue
            c.line(p[prev], p[i], 100)
            rad = 40 if i == ids[-1] else 150
            c.ellipse((p[i][0] - rad, p[i][1] - rad, p[i][0] + rad, p[i][1] + rad))
            prev = i
        clear |= c.m & (labels == label)
    return np.where(clear, 0, labels).astype(np.uint8)


def random_pose(rng, w=768, h=1024):
    """A VITON-HD-like BODY_25 pose on a w x h image (3-decimal coordinates as OpenPose writes them): a jittered upright body; some
    arm joints or hips absent (0, 0), sometimes both hips (the hip rescaling then divides by zero), sometimes joints off the image
    or coincident shoulders."""
    sx, sy = w / 768, h / 1024
    base = np.array([[384, 200], [384, 260], [300, 270], [260, 420], [240, 560], [468, 270], [508, 420], [528, 560], [384, 560],
                     [330, 560], [330, 760], [330, 950], [438, 560], [438, 760], [438, 950]] + [[0, 0]] * 10, float) * [sx, sy]
    p = np.round(base + rng.normal(0, 40 * sx, base.shape), 3)
    p[15:] = 0
    k = rng.integers(0, 8)
    if k == 0:
        p[rng.choice([3, 4, 6, 7], rng.integers(1, 3), replace=False)] = 0
    elif k == 1:
        p[[9, 12]] = 0
    elif k == 2:
        p[rng.choice([2, 3, 5, 6], 1)] += rng.normal(0, 400 * sx, 2)
    elif k == 3:
        p[5] = p[2]
    elif k == 4:
        p[rng.choice([2, 5, 9, 12], 1)] = 0
    return p
