"""A literal restatement, in Python and numpy, of which points indexcov's charts draw (indexcov/plot.go asValues + asPng's
thinning) and of the raster rule plot.cu implements.  numpy's float64 operations round to nearest one at a time, in the
order written here, which is the order the kernel uses, so the images must match bit for bit."""
import numpy as np

CN_MAX = np.float32(2.5)


def as_values(vals, mult):
    """asValues: skip leading values == 0 (NaN is not == 0), x = float64(i) * mult, y = min(v, 2.5)"""
    xs, ys, seen = [], [], False
    for i, r in enumerate(np.asarray(vals, np.float32)):
        if r == 0 and not seen:
            continue
        seen = True
        xs.append(float(i) * mult)
        ys.append(float(CN_MAX if r > CN_MAX else r))
    return xs, ys


def sample(xs, ys):
    """asPng's thinning; None when the dataset is not drawn (NaN left in it)"""
    n = len(xs)
    nth = 10 if n > 2000 else (5 if n > 1000 else 1)
    xs, ys = [x for i, x in enumerate(xs) if i % nth == 0], [y for i, y in enumerate(ys) if i % nth == 0]
    if any(y != y for y in ys):
        return None
    return xs, ys


def select(vals, mult=16384.0):
    """(first, m, stride, ymin, ymax) as gl_plot_select reports them"""
    vals = np.asarray(vals, np.float32)
    nz = np.nonzero(vals != 0)[0]
    first = int(nz[0]) if nz.size else len(vals)
    n = len(vals) - first
    stride = 10 if n > 2000 else (5 if n > 1000 else 1)
    s = sample(*as_values(vals, mult))
    if s is None or not s[0]:
        return first, 0, stride, 0.0, 0.0
    return first, len(s[0]), stride, min(s[1]), max(s[1])


def transform(xmin, xmax, ymin, ymax, W, H):
    if xmin == xmax:
        xmin, xmax = xmin - 1, xmax + 1
    if ymin == ymax:
        ymin, ymax = ymin - 1, ymax + 1
    return np.array([xmin, W / (xmax - xmin), ymin, H / (ymax - ymin)])


def line_radius(n_datasets):
    return max(0.5, (0.65 if n_datasets > 30 else 0.8) * 96.0 / 72.0 / 2.0)


def raster(lines, xf, W, H, r, img=None):
    """lines: [(draw index, xs, ys)] of one chart; the uint32 index image (H, W)"""
    if img is None:
        img = np.zeros((H, W), np.uint32)
    r2 = r * r
    px = np.arange(W, dtype=np.float64) + 0.5
    py = np.arange(H, dtype=np.float64) + 0.5
    PX, PY = np.meshgrid(px, py)
    for idx, xs, ys in lines:
        for j in range(len(xs) - 1):
            ax = (xs[j] - xf[0]) * xf[1]
            ay = float(H) - (ys[j] - xf[2]) * xf[3]
            bx = (xs[j + 1] - xf[0]) * xf[1]
            by = float(H) - (ys[j + 1] - xf[2]) * xf[3]
            dx, dy = bx - ax, by - ay
            L = dx * dx + dy * dy
            ex, ey = PX - ax, PY - ay
            if L != 0.0:
                t = np.clip((ex * dx + ey * dy) / L, 0.0, 1.0)
                qx, qy = ex - t * dx, ey - t * dy
            else:
                qx, qy = ex, ey
            cov = qx * qx + qy * qy <= r2
            img[cov] = np.maximum(img[cov], idx)
    return img


def series_lines(vals_list, mult=16384.0):
    """[(draw index k + 1, xs, ys)] of the drawn datasets, and the chart's (xmin, xmax, ymin, ymax)"""
    lines, ext = [], [np.inf, -np.inf, np.inf, -np.inf]
    for k, v in enumerate(vals_list):
        s = sample(*as_values(v, mult))
        if s is None or not s[0]:
            continue
        xs, ys = s
        lines.append((k + 1, xs, ys))
        ext = [min(ext[0], min(xs)), max(ext[1], max(xs)), min(ext[2], min(ys)), max(ext[3], max(ys))]
    if not lines:
        ext = [0.0, 0.0, 0.0, 0.0]
    return lines, ext
