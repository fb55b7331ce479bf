"""NumPy restatement of the cv2 drawing the reference's report image uses (test infrastructure only, like oracle/jpeg.py),
and of that image's composition (code/utils/utils.py save_correspondences_img + draw_matches).

Every rule below was pinned against cv2 4.13 on the CPU by tests/test_draw_oracle.py (the test that decides each rule is
named in brackets).  Coordinates are Python ints carrying the C integer widths cv2 uses: int32 points, int64 16.16 fixed
point (XY_SHIFT = 16), with two's-complement wrap where cv2's arithmetic wraps.

  polylines(thick 3, LINE_8)   closed: one ThickLine per edge (v[n-1]->v[0], v[0]->v[1], ...), each with an end cap at its
                               second vertex only [test_thick_polyline].  ThickLine = a 4-vertex FillConvexPoly of the
                               segment widened by dp = cvRound((dy, dx) * (thickness/2 + 1/2) / |d|) in 16.16, then the
                               cap: a filled Bresenham circle of radius (thickness*2^15 + 2^15) >> 16 = 2 at the vertex.
  FillConvexPoly(shift 16)     each outline edge drawn with the 16.16 line rasteriser (Line2), then scanlines from the
                               top vertex, edges stepped by dx = ((xe-xs)*2 + (ty-y)) / (2*(ty-y)) (C division) and
                               spans [(xl + 2^15) >> 16, (xr + 2^15) >> 16] clipped to the image [test_fill_convex_poly].
  line(thick 1, LINE_AA)       LineAA on 16.16 points clipped by clipLine to the scaled image: 3 pixels per major step,
                               weights FilterTable x end-point correction, each channel blended twice with
                               v += ((c - v)*a + 127) >> 8 [test_line_aa].  Each step has its own major coordinate, so one
                               segment never visits a pixel twice [test_line_aa_visits_each_pixel_once].
  circle(r, thick 1, LINE_AA)  ellipse2Poly with delta 30 (r = 7 < 10): 13 vertices centre + r*(SinTable[450-a],
                               SinTable[a]), a = 0, 30, ..., 360, each cvRound-ed in two parts (the 16.16 integer part
                               through cvRound(v / 2^16) << 16, then the remainder), repeats dropped, drawn as an open
                               polyline of 12 LineAA segments [test_circle_aa].
  clipping                     clipLine's double-precision intercepts; int32 wrap of the (int) casts cv2 makes, so a
                               vertex at INT_MIN or INT_MAX draws what cv2 draws [test_extreme_vertices].
"""
import math

import numpy as np

XY_SHIFT = 16
XY_ONE = 1 << XY_SHIFT

# The 4.x drawing tables: anti-aliasing filter and slope correction of LineAA, and sin(deg) of ellipse2Poly.
SLOPE_CORR = [181, 181, 181, 182, 182, 183, 184, 185, 187, 188, 190, 192, 194, 196, 198, 201,
              203, 206, 209, 211, 214, 218, 221, 224, 227, 231, 235, 238, 242, 246, 250, 254]
FILTER = [168, 177, 185, 194, 202, 210, 218, 224, 231, 236, 241, 246, 249, 252, 254, 254,
          254, 254, 252, 249, 246, 241, 236, 231, 224, 218, 210, 202, 194, 185, 177, 168,
          158, 149, 140, 131, 122, 114, 105, 97, 89, 82, 75, 68, 62, 56, 50, 45,
          40, 36, 32, 28, 25, 22, 19, 16, 14, 12, 11, 9, 8, 7, 5, 5]

# The report's colours (utils/utils.py:213-217, 263-264), as cv2 receives them: channel 0, 1, 2 of the RGB array.
PRED_COLOR = (5, 225, 225)
GT_COLOR = (2, 10, 240)
MATCH_COLORS = [(255, 102, 255), (51, 153, 255), (102, 255, 255), (255, 255, 0)]


def i32(v):
    return ((v + (1 << 31)) & 0xFFFFFFFF) - (1 << 31)


def i64(v):
    return ((v + (1 << 63)) & 0xFFFFFFFFFFFFFFFF) - (1 << 63)


def cdiv(a, b):
    """C integer division (truncation toward zero)."""
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b >= 0) else -q


def cv_round(x):
    """cvRound(double) on x86-64: round half to even; NaN or outside int32 -> INT_MIN (cvtsd2si)."""
    if not math.isfinite(x):
        return -(1 << 31)
    r = round(x)
    return r if -(1 << 31) <= r < (1 << 31) else -(1 << 31)


def sin_table(deg):
    """OpenCV's SinTable[deg] (float, 7 decimals), deg a multiple of 30 in [0, 450]."""
    return float(np.float32(round(math.sin(math.radians(deg)), 7)))


def clip_line(w, h, x1, y1, x2, y2):
    """clipLine(Size2l, Point2l&, Point2l&) -> (inside, x1, y1, x2, y2).  The second point's intercept uses the first
    point after it was moved, as cv2 does."""
    if w <= 0 or h <= 0:
        return False, x1, y1, x2, y2
    right, bottom = w - 1, h - 1
    c1 = (x1 < 0) + (x1 > right) * 2 + (y1 < 0) * 4 + (y1 > bottom) * 8
    c2 = (x2 < 0) + (x2 > right) * 2 + (y2 < 0) * 4 + (y2 > bottom) * 8
    if (c1 & c2) == 0 and (c1 | c2) != 0:
        if c1 & 12:
            a = 0 if c1 < 8 else bottom
            x1 += int(float(a - y1) * float(x2 - x1) / float(y2 - y1))
            y1 = a
            c1 = (x1 < 0) + (x1 > right) * 2
        if c2 & 12:
            a = 0 if c2 < 8 else bottom
            x2 += int(float(a - y2) * float(x2 - x1) / float(y2 - y1))
            y2 = a
            c2 = (x2 < 0) + (x2 > right) * 2
        if (c1 & c2) == 0 and (c1 | c2) != 0:
            if c1:
                a = 0 if c1 == 1 else right
                y1 += int(float(a - x1) * float(y2 - y1) / float(x2 - x1))
                x1 = a
                c1 = 0
            if c2:
                a = 0 if c2 == 1 else right
                y2 += int(float(a - x2) * float(y2 - y1) / float(x2 - x1))
                x2 = a
                c2 = 0
    return (c1 | c2) == 0, x1, y1, x2, y2


def _put(img, x, y, color):
    img[y, x] = color


def line2(img, x1, y1, x2, y2, color):
    """Line2: the 16.16 LINE_8 rasteriser FillConvexPoly draws its outline with."""
    h, w = img.shape[:2]
    ok, x1, y1, x2, y2 = clip_line(w << XY_SHIFT, h << XY_SHIFT, x1, y1, x2, y2)
    if not ok:
        return
    dx, dy = x2 - x1, y2 - y1
    ax, ay = abs(dx), abs(dy)
    if ax > ay:
        if dx < 0:
            x1, x2, y1, y2, dy = x2, x1, y2, y1, -dy
        xs, ys = XY_ONE, cdiv(dy << XY_SHIFT, ax | 1)
        ecount = (x2 - x1) >> XY_SHIFT
    else:
        if dy < 0:
            x1, x2, y1, y2, dx = x2, x1, y2, y1, -dx
        xs, ys = cdiv(dx << XY_SHIFT, ay | 1), XY_ONE
        ecount = (y2 - y1) >> XY_SHIFT
    x1 += XY_ONE >> 1
    y1 += XY_ONE >> 1
    pts = [(i32((x2 + (XY_ONE >> 1)) >> XY_SHIFT), i32((y2 + (XY_ONE >> 1)) >> XY_SHIFT))]
    for k in range(ecount + 1):
        if ax > ay:
            pts.append((i32((x1 >> XY_SHIFT) + k), i32((y1 + k * ys) >> XY_SHIFT)))
        else:
            pts.append((i32((x1 + k * xs) >> XY_SHIFT), i32((y1 >> XY_SHIFT) + k)))
    for x, y in pts:
        if 0 <= x < w and 0 <= y < h:
            _put(img, x, y, color)


def fill_convex_poly(img, v, color):
    """FillConvexPoly(v in 16.16, LINE_8, shift 16).  Rows between edge events are stepped in closed form (x + k*dx,
    wrapping as cv2's repeated int64 additions do), so far-away vertices cost no time."""
    h, w = img.shape[:2]
    n = len(v)
    delta = XY_ONE >> 1
    px, py = v[n - 1]
    xmin = xmax = v[0][0]
    ymin = ymax = v[0][1]
    imin = 0
    for i, (x, y) in enumerate(v):
        if y < ymin:
            ymin, imin = y, i
        ymax, xmax, xmin = max(ymax, y), max(xmax, x), min(xmin, x)
        line2(img, px, py, x, y, color)
        px, py = x, y
    xmin, xmax = (xmin + delta) >> XY_SHIFT, (xmax + delta) >> XY_SHIFT
    ymin, ymax = (ymin + delta) >> XY_SHIFT, (ymax + delta) >> XY_SHIFT
    if n < 3 or i32(xmax) < 0 or i32(ymax) < 0 or i32(xmin) >= w or i32(ymin) >= h:
        return
    ymax = min(ymax, h - 1)
    ylast = i32(ymax)
    edges = n
    # edge: [idx, di, x, dx, ye]
    e = [[imin, 1, -XY_ONE, 0, i32(ymin)], [imin, n - 1, -XY_ONE, 0, i32(ymin)]]
    y = i32(ymin)
    while True:
        for i in range(2):
            if y >= e[i][4]:
                idx0, di = e[i][0], e[i][1]
                idx = idx0 + di
                if idx >= n:
                    idx -= n
                while True:
                    edges -= 1
                    if edges + 1 <= 0:
                        break
                    ty = i32((v[idx][1] + delta) >> XY_SHIFT)
                    if ty > y:
                        xs, xe = v[idx0][0], v[idx][0]
                        e[i][4] = ty
                        e[i][3] = cdiv((xe - xs) * 2 + (ty - y), 2 * (ty - y))
                        e[i][2] = xs
                        e[i][0] = idx
                        break
                    idx0 = idx
                    idx += di
                    if idx >= n:
                        idx -= n
        if edges < 0:
            return
        stop = min(e[0][4], e[1][4], ylast + 1)
        for r in range(max(y, 0), stop):
            k = r - y
            x0, x1 = i64(e[0][2] + k * e[0][3]), i64(e[1][2] + k * e[1][3])
            left, right = (x1, x0) if x0 > x1 else (x0, x1)
            xx1 = i32(i64(left + delta) >> XY_SHIFT)
            xx2 = i32(i64(right + delta) >> XY_SHIFT)
            if xx2 >= 0 and xx1 < w:
                img[r, max(xx1, 0):min(xx2, w - 1) + 1] = color
        for i in range(2):
            e[i][2] = i64(e[i][2] + (stop - y) * e[i][3])
        y = stop
        if y > ylast:
            return


def circle_fill(img, cx, cy, r, color):
    """Circle(fill = 1): Bresenham spans, int32 wrap in the span ends."""
    h, w = img.shape[:2]
    err, dx, dy, plus, minus = 0, r, 0, 1, (r << 1) - 1
    while dx >= dy:
        y11, y12, y21, y22 = i32(cy - dy), i32(cy + dy), i32(cy - dx), i32(cy + dx)
        x11, x12, x21, x22 = i32(cx - dx), i32(cx + dx), i32(cx - dy), i32(cx + dy)
        if x11 < w and x12 >= 0 and y21 < h and y22 >= 0:
            x11, x12 = max(x11, 0), min(x12, w - 1)
            for yy in (y11, y12):
                if 0 <= yy < h:
                    img[yy, x11:x12 + 1] = color
            if x21 < w and x22 >= 0:
                x21, x22 = max(x21, 0), min(x22, w - 1)
                for yy in (y21, y22):
                    if 0 <= yy < h:
                        img[yy, x21:x22 + 1] = color
        dy += 1
        err += plus
        plus += 2
        mask = 0 if err <= 0 else -1
        err -= minus & mask
        dx += mask
        minus -= mask & 2


def line_aa_pixels(w, h, x1, y1, x2, y2):
    """LineAA on 16.16 points -> the (x, y, a) it blends, in cv2's order."""
    ok, x1, y1, x2, y2 = clip_line(w << XY_SHIFT, h << XY_SHIFT, x1, y1, x2, y2)
    if not ok:
        return []
    dx, dy = x2 - x1, y2 - y1
    ax, ay = abs(dx), abs(dy)
    horiz = ax > ay
    if horiz:
        if dx < 0:
            x1, x2, y1, y2, dy = x2, x1, y2, y1, -dy
        step = cdiv(dy << XY_SHIFT, ax | 1)
        x2 += XY_ONE
        ecount = (x2 >> XY_SHIFT) - (x1 >> XY_SHIFT)
        j = -(x1 & (XY_ONE - 1))
        y1 += ((step * j) >> XY_SHIFT) + (XY_ONE >> 1)
        fi, fj = (x1 >> (XY_SHIFT - 7)) & 0x78, (x2 >> (XY_SHIFT - 7)) & 0x78
        major, minor = x1 >> XY_SHIFT, y1
    else:
        if dy < 0:
            x1, x2, y1, y2, dx = x2, x1, y2, y1, -dx
        step = cdiv(dx << XY_SHIFT, ay | 1)
        y2 += XY_ONE
        ecount = (y2 >> XY_SHIFT) - (y1 >> XY_SHIFT)
        j = -(y1 & (XY_ONE - 1))
        x1 += ((step * j) >> XY_SHIFT) + (XY_ONE >> 1)
        fi, fj = (y1 >> (XY_SHIFT - 7)) & 0x78, (y2 >> (XY_SHIFT - 7)) & 0x78
        major, minor = y1 >> XY_SHIFT, x1
    slope = (step >> (XY_SHIFT - 5)) & 0x3F
    slope ^= 0x3F if step < 0 else 0
    slope = 0x100 if slope & 0x20 else SLOPE_CORR[slope]
    t0, t1, t2 = slope << 7, ((0x78 - fi) | 4) * slope, (fj | 4) * slope
    ep = [0, 0, (t1 >> 8) & 0x1FF, 0, ((((fj - fi) + 0x80) | 4) * slope >> 8) & 0x1FF, ((t1 + t0) >> 8) & 0x1FF,
          (t2 >> 8) & 0x1FF, ((t2 + t0) >> 8) & 0x1FF, slope]
    ep[1] = ep[3] = ((((fj - fi) & 0x78) | 4) * slope >> 8) & 0x1FF
    size_major, size_minor = (w, h) if horiz else (h, w)
    out = []
    for s in range(ecount + 1):
        ec = ecount - s
        m = i32(major + s)
        if not 0 <= m < size_major:
            continue
        pos = minor + s * step
        q = i32((pos >> XY_SHIFT) - 1)
        corr = ep[(((s >= 2) + 1) & (s | 2)) * 3 + (((ec >= 2) + 1) & (ec | 2))]
        dist = (pos >> (XY_SHIFT - 5)) & 31
        for o, f in ((0, FILTER[dist + 32]), (1, FILTER[dist]), (2, FILTER[63 - dist])):
            if 0 <= q + o < size_minor:
                a = (corr * f >> 8) & 0xFF
                out.append((m, q + o, a) if horiz else (q + o, m, a))
    return out


def blend(v, c, a):
    v += ((c - v) * a + 127) >> 8
    v += ((c - v) * a + 127) >> 8
    return v


def line_aa(img, x1, y1, x2, y2, color):
    h, w = img.shape[:2]
    for x, y, a in line_aa_pixels(w, h, x1, y1, x2, y2):
        px = img[y, x]
        img[y, x] = [blend(int(px[c]), color[c], a) for c in range(3)]


def clip_thick(w, h, m, p0, p1):
    """A thick segment is first clipped, on int32 points, to the image grown by m = thickness on every side (so a
    clipped end and its cap lie outside the image)."""
    ok, x0, y0, x1, y1 = clip_line(w + 2 * m, h + 2 * m, p0[0] + m, p0[1] + m, p1[0] + m, p1[1] + m)
    return ok, (x0 - m, y0 - m), (x1 - m, y1 - m)


def thick_line(img, p0, p1, color, thickness, aa, flags):
    """ThickLine(shift 0) on int32 points."""
    if thickness <= 1:
        assert aa, "only the LINE_AA thin line and the thick LINE_8 line are used"
        line_aa(img, p0[0] << XY_SHIFT, p0[1] << XY_SHIFT, p1[0] << XY_SHIFT, p1[1] << XY_SHIFT, color)
        return
    h, w = img.shape[:2]
    ok, p0, p1 = clip_thick(w, h, thickness, p0, p1)
    if not ok:
        return
    x0, y0, x1, y1 = p0[0] << XY_SHIFT, p0[1] << XY_SHIFT, p1[0] << XY_SHIFT, p1[1] << XY_SHIFT
    dxf, dyf = (x0 - x1) / XY_ONE, (y1 - y0) / XY_ONE
    r = dxf * dxf + dyf * dyf
    odd = thickness & 1
    th = thickness << (XY_SHIFT - 1)
    if abs(r) > 2.220446049250313e-16:
        r = (th + odd * XY_ONE * 0.5) / math.sqrt(r)
        dpx, dpy = cv_round(dyf * r), cv_round(dxf * r)
        fill_convex_poly(img, [(x0 + dpx, y0 + dpy), (x0 - dpx, y0 - dpy), (x1 - dpx, y1 - dpy), (x1 + dpx, y1 + dpy)], color)
    for i, (x, y) in enumerate(((x0, y0), (x1, y1))):
        if flags & (i + 1):
            circle_fill(img, i32((x + (XY_ONE >> 1)) >> XY_SHIFT), i32((y + (XY_ONE >> 1)) >> XY_SHIFT),
                        (th + (XY_ONE >> 1)) >> XY_SHIFT, color)


def polylines_closed(img, pts, color, thickness=3):
    """cv2.polylines(img, [pts], True, color, thickness) with LINE_8, pts int32 [n,2]."""
    pts = [(int(x), int(y)) for x, y in pts]
    p0 = pts[-1]
    for p in pts:
        thick_line(img, p0, p, color, thickness, False, 2)
        p0 = p


def line(img, p0, p1, color):
    """cv2.line(img, p0, p1, color, 1, LINE_AA)."""
    thick_line(img, (int(p0[0]), int(p0[1])), (int(p1[0]), int(p1[1])), color, 1, True, 3)


def circle_poly(cx, cy, r):
    """EllipseEx's 16.16 polygon of cv2.circle(centre, r, thickness 1, LINE_AA) for r in [3, 10)."""
    cxd, cyd, ad = float(cx << XY_SHIFT), float(cy << XY_SHIFT), float(r << XY_SHIFT)
    v = []
    for ang in range(0, 390, 30):
        x, y = ad * sin_table(450 - ang), ad * sin_table(ang)
        fx, fy = cxd + x * 1.0 - y * 0.0, cyd + x * 0.0 + y * 1.0
        pt = []
        for f in (fx, fy):
            q = cv_round(f / XY_ONE) << XY_SHIFT
            pt.append(q + cv_round(f - q))
        if not v or tuple(pt) != v[-1]:
            v.append(tuple(pt))
    return v


def circle(img, c, r, color):
    """cv2.circle(img, c, r, color, 1, LINE_AA)."""
    assert 3 <= r < 10
    v = circle_poly(int(c[0]), int(c[1]), r)
    for a, b in zip(v[:-1], v[1:]):
        line_aa(img, a[0], a[1], b[0], b[1], color)


# ---------------------------------------------------------------------------------------------------- the report
EXTREMES = [30000, 40000, 1 << 20, (1 << 31) - 1, -(1 << 31), -30000, -40000, -(1 << 20)]


def vertex_cases(rng, n, h, w):
    """n seeded report vertex sets [n,20,2] int32 for images h x w (canvas h x 2w), cycling through: anywhere on the
    canvas (all octants), on / just outside the border, horizontal / vertical / 45-degree edges, zero-length lines and
    coincident vertices, far outside, and the int32 extremes (INT_MIN is what np.int32(nan) gives)."""
    out = np.empty((n, 20, 2), np.int64)
    dirs = np.array([(1, 0), (0, 1), (1, 1), (1, -1), (-1, 0), (0, -1), (-1, -1), (-1, 1)])
    for k in range(n):
        kind = k % 6
        v = np.stack([rng.integers(-8, 2 * w + 8, 20), rng.integers(-8, h + 8, 20)], 1)
        if kind == 1:
            v[:, 0] = rng.choice([-3, -2, -1, 0, 1, w - 1, w, 2 * w - 2, 2 * w - 1, 2 * w, 2 * w + 2], 20)
            v[:, 1] = np.where(rng.random(20) < 0.5, rng.choice([-3, -1, 0, 1, h - 2, h - 1, h, h + 2], 20), v[:, 1])
        elif kind == 2:
            for s in (0, 4, 8):
                for j in range(1, 4):
                    v[s + j] = v[s + j - 1] + rng.integers(1, 2 * w) * dirs[rng.integers(0, 8)]
            for i in range(4):
                v[16 + i] = v[12 + i] + rng.integers(1, 2 * w) * dirs[rng.integers(0, 8)]
        elif kind == 3:
            m = rng.random(20) < 0.5
            v[m] = v[np.maximum(np.flatnonzero(m) - 1, 0)]
            z = rng.random(4) < 0.5
            v[16:20][z] = v[12:16][z]
        elif kind == 4:
            v = v + rng.choice([-1, 1], (20, 2)) * rng.integers(100, 5000, (20, 2)) * (rng.random((20, 1)) < 0.4)
        elif kind == 5:
            m = rng.random((20, 2)) < 0.25
            v[m] = rng.choice(EXTREMES, int(m.sum()))
        out[k] = v
    return out.astype(np.int32)


def draw_report(img1, img2, verts):
    """The report canvas [h, w1+w2, 3] from the two uint8 images and the int32 vertices [20,2]: prediction polygon
    (right-image coordinates), kp2, kp1, match line starts, match line ends."""
    img2 = img2.copy()
    polylines_closed(img2, verts[0:4], PRED_COLOR)                           # drawn on img2 alone, before stacking
    h, w1 = img1.shape[:2]
    canvas = np.zeros((h, w1 + img2.shape[1], 3), np.uint8)
    canvas[:, :w1] = img1
    canvas[:, w1:] = img2
    polylines_closed(canvas, verts[4:8], GT_COLOR)
    polylines_closed(canvas, verts[8:12], GT_COLOR)
    for i in range(4):
        line(canvas, verts[12 + i], verts[16 + i], MATCH_COLORS[i])
        circle(canvas, verts[12 + i], 7, MATCH_COLORS[i])
        circle(canvas, verts[16 + i], 7, MATCH_COLORS[i])
    return canvas


def cv2_draw_report(img1, img2, verts):
    """The same drawing as the cv2 call sequence of utils/utils.py:209-296 (cv2 imported here: the tests' oracle)."""
    import cv2
    v = [tuple(int(c) for c in p) for p in verts]
    img2 = img2.copy()
    cv2.polylines(img2, np.int32([v[0:4]]), 1, PRED_COLOR, 3)
    h, w1 = img1.shape[:2]
    out = np.zeros((h, w1 + img2.shape[1], 3), np.uint8)
    out[:, :w1] = img1
    out[:, w1:] = img2
    cv2.polylines(out, np.int32([v[4:8]]), 1, GT_COLOR, 3)
    cv2.polylines(out, np.int32([v[8:12]]), 1, GT_COLOR, 3)
    for i in range(4):
        cv2.line(out, v[12 + i], v[16 + i], MATCH_COLORS[i], 1, cv2.LINE_AA)
        cv2.circle(out, v[12 + i], 7, MATCH_COLORS[i], 1, cv2.LINE_AA)
        cv2.circle(out, v[16 + i], 7, MATCH_COLORS[i], 1, cv2.LINE_AA)
    return out


def cv2_compose(img1, img2, corr1, corr2, pred_corr2):
    """save_correspondences_img from the float points, with the reference's own conversions (utils/utils.py:209-296)."""
    import cv2
    img2 = img2.copy()
    cv2.polylines(img2, np.int32([pred_corr2]), 1, PRED_COLOR, 3)
    h, w1 = img1.shape[:2]
    out = np.zeros((h, w1 + img2.shape[1], 3), np.uint8)
    out[:, :w1] = img1
    out[:, w1:] = img2
    kp2 = (corr2 + np.array([w1, 0])).astype(np.int32)
    kp1 = corr1.astype(np.int32)
    cv2.polylines(out, np.int32([kp2]), 1, GT_COLOR, 3)
    cv2.polylines(out, np.int32([kp1]), 1, GT_COLOR, 3)
    for i in range(4):
        end1 = tuple(int(c) for c in np.round(kp1[i]).astype(int))
        end2 = tuple(int(c) for c in np.round(corr2[i]).astype(int) + np.array([w1, 0]))
        cv2.line(out, end1, end2, MATCH_COLORS[i], 1, cv2.LINE_AA)
        cv2.circle(out, end1, 7, MATCH_COLORS[i], 1, cv2.LINE_AA)
        cv2.circle(out, end2, 7, MATCH_COLORS[i], 1, cv2.LINE_AA)
    return out


MEAN32, STD32 = np.float32([118.93, 113.97, 102.60]), np.float32([69.85, 68.81, 72.45])
MEAN64, STD64 = np.float64([118.93, 113.97, 102.60]), np.float64([69.85, 68.81, 72.45])


def host_denorm(u8, aug_row=None, im=0):
    """denorm_img(normalise(augment(I))).astype(uint8) on the host (utils/utils.py:406-413), image im (0: I, 1: I') of
    a [11] augmentation row as udh_prep_inputs_u8_ex reads it (flag, then gamma, brightness, 3 colour gains per image):
    pow in float64 rounded once to float32, then the float32 products, clip, normalise; float64 denorm, truncation."""
    v = u8.astype(np.float32)
    if aug_row is not None and aug_row[0] != 0:
        a = np.asarray(aug_row, np.float32)[1 + 5 * im:6 + 5 * im]
        v = np.power(u8.astype(np.float64), np.float64(a[0])).astype(np.float32)
        v = (v * a[1]).astype(np.float32)
        v = (v * a[2:5]).astype(np.float32)
        v = np.clip(v, np.float32(0), np.float32(255))
    n = ((v - MEAN32) / STD32).astype(np.float32)
    return np.clip(np.trunc(n.astype(np.float64) * STD64 + MEAN64), 0, 255).astype(np.uint8)
