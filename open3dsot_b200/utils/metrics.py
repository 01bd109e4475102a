"""Tracking metrics with the reference's names and definitions (utils/metrics.py:27-128): `estimateOverlap` (bird's-eye
or 3-D IoU of two boxes), `estimateAccuracy` (centre distance), and the Success / Precision curves' areas.
shapely / torchmetrics are replaced by a half-plane clip of the two convex footprints and plain accumulators."""
import numpy as np

_trapz = getattr(np, "trapezoid", None) or np.trapz   # numpy >= 2.0 renamed trapz


def estimateAccuracy(box_a, box_b, dim=3, up_axis=(0, -1, 0)):
    if dim == 3:
        return float(np.linalg.norm(box_a.center - box_b.center, ord=2))
    keep = np.array(up_axis) != 0
    return float(np.linalg.norm(box_a.center[keep] - box_b.center[keep], ord=2))


def _footprint(box, up_axis):
    """The quadrilateral the reference hands to shapely (fromBoxToPoly :37-47), as (4, 2), counter-clockwise."""
    if up_axis[1] != 0:
        poly = box.corners()[[0, 2]].T[[0, 1, 5, 4]]
    else:
        poly = box.bottom_corners().T[:, :2]
    x, y = poly[:, 0], poly[:, 1]
    signed = np.dot(x, np.roll(y, -1)) - np.dot(y, np.roll(x, -1))
    return poly if signed > 0 else poly[::-1]


def _poly_area(p):
    if len(p) < 3:
        return 0.0
    return 0.5 * abs(np.dot(p[:, 0], np.roll(p[:, 1], -1)) - np.dot(p[:, 1], np.roll(p[:, 0], -1)))


def _intersection_area(pa, pb):
    """Area of the intersection of two convex counter-clockwise polygons: `pa` clipped by each edge half-plane of `pb`."""
    poly = pa
    for i in range(len(pb)):
        if len(poly) == 0:
            return 0.0
        a, e = pb[i], pb[(i + 1) % len(pb)] - pb[i]
        side = e[0] * (poly[:, 1] - a[1]) - e[1] * (poly[:, 0] - a[0])       # >= 0: inside
        nxt, side_n = np.roll(poly, -1, axis=0), np.roll(side, -1)
        out = []
        for p, q, s, t in zip(poly, nxt, side, side_n):
            if s >= 0:
                out.append(p)
            if (s >= 0) != (t >= 0):
                out.append(p + (q - p) * (s / (s - t)))
        poly = np.array(out).reshape(-1, 2)
    return _poly_area(poly)


def estimateOverlap(box_a, box_b, dim=2, up_axis=(0, -1, 0), footprints=None):
    """`footprints`: the boxes' `_footprint`s when the caller already has them (one per box, not one per pair)."""
    pa, pb = footprints if footprints is not None else (_footprint(box_a, up_axis), _footprint(box_b, up_axis))
    inter = _intersection_area(pa, pb)
    if dim == 2:
        union = _poly_area(pa) + _poly_area(pb) - inter
        return float(inter / union) if union > 0 else 0.0
    up = np.array(up_axis) != 0
    up_max = min(box_a.center[up], box_b.center[up])
    up_min = max(box_a.center[up] - box_a.wlh[2], box_b.center[up] - box_b.wlh[2])
    inter_vol = inter * max(0.0, float(up_max[0] - up_min[0]))
    va, vb = float(np.prod(box_a.wlh)), float(np.prod(box_b.wlh))
    return float(inter_vol / (va + vb - inter_vol))


class _Curve:
    def __init__(self, n, top):
        self.top, self.xs, self.vals = top, np.linspace(0, top, n), []

    def update(self, val):
        self.vals.extend(np.atleast_1d(np.asarray(val, dtype=np.float64)).tolist())

    __call__ = update

    def reset(self):
        self.vals = []


class Success(_Curve):
    """TorchSuccess (:104-128): area under fraction(overlap >= t), t in [0, max_overlap], in percent."""

    def __init__(self, n=21, max_overlap=1):
        super().__init__(n, max_overlap)

    def compute(self):
        if not self.vals:
            return 0.0
        v = np.asarray(self.vals)
        return float(_trapz([(v >= t).mean() for t in self.xs], self.xs) * 100 / self.top)


class Precision(_Curve):
    """TorchPrecision (:77-101): area under fraction(distance <= t), t in [0, max_accuracy], in percent."""

    def __init__(self, n=21, max_accuracy=2):
        super().__init__(n, max_accuracy)

    def compute(self):
        if not self.vals:
            return 0.0
        v = np.asarray(self.vals)
        return float(_trapz([(v <= t).mean() for t in self.xs], self.xs) * 100 / self.top)
