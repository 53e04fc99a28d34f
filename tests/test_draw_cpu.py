"""CPU: the rasterisation rules of csrc/draw_kernels.cu, stated in numpy (draw_oracle), against ImageDraw itself on seeded random
shapes, and the restated get_agnostic / get_parse_agnostic against data.agnostic_bits and the reference's get_im_parse_agnostic.
No tolerance: a mask pixel matches or it does not."""
import os
import sys

import numpy as np
import pytest
from PIL import Image, ImageDraw

import hrv_env
from hrviton_b200 import data, draw

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import draw_oracle as O  # noqa: E402


def _coord(rng, lo, hi):
    """Integral, half-integral or arbitrary fractional coordinates, negative ones and ones past the canvas included."""
    v = rng.uniform(lo, hi)
    k = rng.integers(0, 3)
    return float(np.round(v)) if k == 0 else float(np.round(v * 2) / 2) if k == 1 else float(v)


def _pil(w, h, fn):
    im = Image.new("L", (w, h), 0)
    fn(ImageDraw.Draw(im))
    return np.asarray(im) != 0


def _canvas(rng):
    return int(rng.integers(1, 40)), int(rng.integers(1, 40))


def test_ellipse_matches_imagedraw():
    rng = np.random.default_rng(1)
    for _ in range(3000):
        w, h = _canvas(rng)
        x0, y0 = _coord(rng, -12, w + 6), _coord(rng, -12, h + 6)
        k = rng.integers(0, 4)  # degenerate extents (0 - 2 px) in x, y, both, or neither
        ex = _coord(rng, 0, 2) if k in (0, 2) else _coord(rng, 0, 30)
        ey = _coord(rng, 0, 2) if k in (1, 2) else _coord(rng, 0, 30)
        box = (x0, y0, x0 + ex, y0 + ey)
        c = O.Canvas(w, h)
        c.ellipse(box)
        assert np.array_equal(c.m, _pil(w, h, lambda d: d.ellipse(box, 255, 255))), (w, h, box)


def test_rectangle_matches_imagedraw():
    rng = np.random.default_rng(2)
    for _ in range(2000):
        w, h = _canvas(rng)
        x0, y0 = _coord(rng, -12, w + 6), _coord(rng, -12, h + 6)
        box = (x0, y0, x0 + _coord(rng, 0, 30), y0 + _coord(rng, 0, 30))
        c = O.Canvas(w, h)
        c.rectangle(box)
        assert np.array_equal(c.m, _pil(w, h, lambda d: d.rectangle(box, 255, 255))), (w, h, box)


def test_line_matches_imagedraw():
    rng = np.random.default_rng(3)
    for t in range(4000):
        w, h = _canvas(rng)
        p = (_coord(rng, -15, w + 15), _coord(rng, -15, h + 15))
        k = t % 5  # zero-length, near-vertical, near-horizontal, arbitrary (twice)
        q = (p if k == 0 else (p[0] + _coord(rng, -1, 1), p[1] + _coord(rng, -30, 30)) if k == 1 else
             (p[0] + _coord(rng, -30, 30), p[1] + _coord(rng, -1, 1)) if k == 2 else (_coord(rng, -15, w + 15), _coord(rng, -15, h + 15)))
        width = int(rng.integers(0, 26))  # <= 1 (Bresenham), even and odd
        c = O.Canvas(w, h)
        c.line(p, q, width)
        assert np.array_equal(c.m, _pil(w, h, lambda d: d.line([p, q], 255, width=width))), (w, h, p, q, width)


def _convex_after_truncation(pts, min_angle=15.0):
    """The truncated vertices form a convex polygon whose corners (collinear vertices aside) are at least min_angle degrees."""
    v = [(O.cint(x), O.cint(y)) for x, y in pts]
    v = [a for i, a in enumerate(v) if a != v[i - 1]]
    sign, corners = 0, 0
    for i in range(len(v)):
        (ax, ay), (bx, by), (cx, cy) = v[i - 2], v[i - 1], v[i]
        cr = (bx - ax) * (cy - by) - (by - ay) * (cx - bx)
        if cr:
            if sign and (cr > 0) != (sign > 0):
                return False
            sign = cr
            corners += 1
            u, t = np.array([ax - bx, ay - by], float), np.array([cx - bx, cy - by], float)
            if np.degrees(np.arccos(np.clip(u @ t / np.linalg.norm(u) / np.linalg.norm(t), -1, 1))) < min_angle:
                return False
    return corners >= 3


def test_polygon_matches_imagedraw():
    """Convex polygons (as their truncated vertices are) with no corner sharper than 15 degrees, with coincident and collinear
    vertices, in either orientation: the class of get_agnostic's torso quadrilateral.  (Wide lines' polygons, rectangles of any
    aspect, are covered by test_line_matches_imagedraw.)  draw.c's rule for sharp corners is not fully restated: on thin slivers
    and self-intersecting polygons the restatement can differ from ImageDraw at the spike's tip."""
    from scipy.spatial import ConvexHull
    rng = np.random.default_rng(4)
    done = 0
    while done < 2000:
        w, h = _canvas(rng)
        pts = rng.uniform(-10, [w + 10, h + 10], (int(rng.integers(3, 8)), 2))
        if rng.integers(0, 2):
            pts = np.round(pts * 2) / 2
        try:
            pts = [tuple(map(float, p)) for p in pts[ConvexHull(pts).vertices]]
        except Exception:  # noqa: BLE001  (flat point sets)
            continue
        if rng.integers(0, 3) == 0:
            pts.insert(1, pts[0])  # coincident
        if rng.integers(0, 3) == 0:
            a, b, s = pts[-1], pts[0], rng.uniform(0, 1)
            pts.append((a[0] + (b[0] - a[0]) * s, a[1] + (b[1] - a[1]) * s))  # collinear
        if rng.integers(0, 2):
            pts = pts[::-1]
        if not _convex_after_truncation(pts):
            continue
        c = O.Canvas(w, h)
        c.polygon(pts)
        assert np.array_equal(c.m, _pil(w, h, lambda d: d.polygon(pts, 255, 255))), (w, h, pts)
        done += 1


def test_restated_agnostic_bits_match_data():
    rng = np.random.default_rng(5)
    for _ in range(200):
        pose = O.random_pose(rng)
        with np.errstate(all="ignore"):  # both hips absent: the reference divides 0 by 0 and draws NaN shapes
            want = data.agnostic_bits(pose, data.ARM_CANVAS)
        assert np.array_equal(O.agnostic_bits(pose), want), pose.tolist()


def _labels(rng, h, w, pose):
    lab = np.kron(rng.integers(0, 20, (h // 32 + 1, w // 32 + 1)), np.ones((32, 32), np.int64))[:h, :w].astype(np.uint8)
    im = Image.fromarray(lab, "L")
    d = ImageDraw.Draw(im)
    for label, joints in ((14, (5, 6, 7)), (15, (2, 3, 4))):
        d.line([tuple(pose[j]) for j in joints], label, width=60)
    return np.asarray(im)


@pytest.fixture(scope="module")
def ref_parse():
    if hrv_env.reference_dir() is None:
        pytest.skip("no reference copy (oracle/_ref)")
    return hrv_env.load_reference_script("get_parse_agnostic")


def test_restated_parse_agnostic_matches_reference(ref_parse):
    rng = np.random.default_rng(6)
    for i in range(24):
        h, w = (1024, 768) if i % 3 else (512, 384)
        pose = O.random_pose(rng, w, h)
        lab = _labels(rng, h, w, pose)
        want = np.asarray(ref_parse.get_im_parse_agnostic(Image.fromarray(lab, "L"), pose.copy(), w=w, h=h))
        assert np.array_equal(O.parse_agnostic(lab, pose), want), i


def test_golden_fixture_matches_restatement(golden_dir):
    g = np.load(os.path.join(golden_dir, "parse_agnostic_512x384_b6.npz"))
    for lab, kp, want in zip(g["labels"], g["keypoints"], g["result"]):
        assert np.array_equal(O.parse_agnostic(lab, kp), want)


def test_write_png_is_the_reference_file(ref_parse, tmp_path):
    """The tool's writer (source mode, palette and info; PIL's save) gives the reference script's bytes for the same labels."""
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
    import parse_agnostic as tool
    rng = np.random.default_rng(7)
    for mode in ("P", "L"):
        pose = O.random_pose(rng)
        im = Image.fromarray(_labels(rng, 1024, 768, pose), mode)
        if mode == "P":
            im.putpalette([int(v) for v in rng.integers(0, 256, 768)])
        src = str(tmp_path / ("src_%s.png" % mode))
        im.save(src)
        ref_out, out = str(tmp_path / "ref.png"), str(tmp_path / "out.png")
        ref_parse.get_im_parse_agnostic(Image.open(src), pose.copy()).save(ref_out)
        tool.write_png(src, O.parse_agnostic(np.asarray(Image.open(src)), pose), out)
        with open(ref_out, "rb") as a, open(out, "rb") as b:
            assert a.read() == b.read(), mode


def test_keypoints_array_refusals():
    ok = np.zeros((25, 2))
    assert draw.keypoints_array(ok).shape == (25, 2)
    assert np.array_equal(draw.keypoints_array(np.ones((18, 2)))[18:], np.zeros((7, 2)))  # COCO-18: the rest absent
    for bad in (np.zeros((12, 2)), np.zeros((25, 3)), np.full((25, 2), np.nan), np.full((25, 2), 5000.0)):
        with pytest.raises(ValueError):
            draw.keypoints_array(bad, "x.json")
