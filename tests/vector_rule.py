"""A restatement, in Python, of the vector charts' path text (INDEXCOV_FMT; plot.cu): each vertex at
Xpt = 0.75 * (AX + (x - xmin) * sx), Ypt = 0.75 * (AY + (H - (y - ymin) * sy)) (EPS: 0.75 * CH - Ypt), every operation one
float64 step in that order, written as "%.2f" of the float64 value.  Python's float arithmetic and "%" formatting are
IEEE float64 and exact decimal rounding, so the bytes must match."""
import math
import re

AX, AY = 56, 8
CANVAS = {0: (316, 244, 384, 288), 1: (316, 244, 384, 288), 2: (508, 532, 576, 576)}   # kind: W, H, CW, CH in pixels
SVG, EPS = 0, 1


def point(x, y, xf, kind, fmt):
    H, CH = CANVAS[kind][1], CANVAS[kind][3]
    X = 0.75 * (AX + (x - xf[0]) * xf[1])
    Y = 0.75 * (AY + (H - (y - xf[2]) * xf[3]))
    if fmt == EPS:
        Y = 0.75 * CH - Y
    return X, Y


def path_text(xs, ys, xf, kind, fmt):
    """the path text of one dataset (b"" when it is not written)"""
    if len(xs) < 2:
        return b""
    out = []
    for j, (x, y) in enumerate(zip(xs, ys)):
        X, Y = point(x, y, xf, kind, fmt)
        if not (math.isfinite(X) and math.isfinite(Y)) or max(abs(X), abs(Y)) >= 1e12:
            return b""
        if fmt == SVG:
            out.append(("M " if j == 0 else " L ") + "%.2f %.2f" % (X, Y))
        else:
            out.append("%.2f %.2f %s\n" % (X, Y, "moveto" if j == 0 else "lineto"))
    return "".join(out).encode()


_NUM = r"-?\d+\.\d\d"


def parse_path(text, fmt):
    """[(X, Y)] as the strings of the path text, checking its grammar on the way"""
    text = text.decode() if isinstance(text, bytes) else text
    if fmt == SVG:
        m = re.fullmatch(r"M (%s) (%s)((?: L %s %s)*)" % (_NUM, _NUM, _NUM, _NUM), text)
        assert m, text[:200]
        return [(m.group(1), m.group(2))] + re.findall(r" L (%s) (%s)" % (_NUM, _NUM), m.group(3))
    lines = text.split("\n")
    assert lines[-1] == ""
    pts = []
    for j, ln in enumerate(lines[:-1]):
        m = re.fullmatch(r"(%s) (%s) (moveto|lineto)" % (_NUM, _NUM), ln)
        assert m and m.group(3) == ("moveto" if j == 0 else "lineto"), ln
        pts.append((m.group(1), m.group(2)))
    return pts
