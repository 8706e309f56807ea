"""An independent restatement of the top-level rule of raytracing_b200/csrc/rt_instances.h (include/rt_b200.h, instanced scenes),
written from the stated rule with numpy: W = adj(A) / det and -(W t) in double rounded to float, world boxes from the 8 transformed corners in
double, padded by 2^-20 of their largest magnitude and rounded outward to float, the median split on the longest centroid axis
with records in depth-first preorder, and the slack (a, b) by which the traversal widens every top-level box."""
import numpy as np

PAD = 2.0 ** -20


SLACK = 2.0 ** -16


def inverse(m):
    """(W as float32 (3, 4), sign of det) of a row-major 3x4 matrix, or None when it is not finite or singular."""
    r = _inverse(m)
    return None if r is None else r[:2]


def _inverse(m):
    """-> (W float32, sign, kappa = ||A||_inf ||A^-1||_inf in double), or None."""
    m = np.asarray(m, np.float32).astype(np.float64).reshape(3, 4)
    if not np.all(np.isfinite(m)):
        return None
    a = m[:, :3]
    det = (a[0, 0] * (a[1, 1] * a[2, 2] - a[1, 2] * a[2, 1]) - a[0, 1] * (a[1, 0] * a[2, 2] - a[1, 2] * a[2, 0])
           + a[0, 2] * (a[1, 0] * a[2, 1] - a[1, 1] * a[2, 0]))
    if det == 0.0 or not np.isfinite(det):
        return None
    (a_, b, c), (d, e, f), (g, h, k) = a
    inv = np.array([[e * k - f * h, c * h - b * k, b * f - c * e],           # adj(A) / det, each entry divided in double
                    [f * g - d * k, a_ * k - c * g, c * d - a_ * f],
                    [d * h - e * g, b * g - a_ * h, a_ * e - b * d]]) / det
    w = np.zeros((3, 4))
    w[:, :3] = inv
    t = m[:, 3]
    w[:, 3] = -((inv[:, 0] * t[0] + inv[:, 1] * t[1]) + inv[:, 2] * t[2])
    norm = lambda x: max((abs(x[r, 0]) + abs(x[r, 1])) + abs(x[r, 2]) for r in range(3))
    return w.astype(np.float32), (-1.0 if det < 0 else 1.0), norm(a) * norm(inv)


def slack(mats, boxes):
    """The header's (a, b) over instances with matrices mats (n, 3, 4) and world boxes (n, 6): a = 2^-16 max kappa_i, b = 2^-16
    max kappa_i (s_i + |t_i|_inf), s_i the largest |coordinate| of box i, t_i the translation; rounded up to float."""
    a = b = 0.0
    for m, box in zip(mats, boxes):
        kappa = _inverse(m)[2]
        s = float(np.abs(np.asarray(box, np.float64)).max())
        t = float(np.abs(np.asarray(m, np.float32).reshape(3, 4)[:, 3].astype(np.float64)).max())
        a, b = max(a, kappa), max(b, kappa * (s + t))
    return np.array([_up(SLACK * a), _up(SLACK * b)], np.float32)


def _down(v):
    f = np.float32(v)
    return np.nextafter(f, np.float32(-np.inf)) if float(f) > v else f


def _up(v):
    f = np.float32(v)
    return np.nextafter(f, np.float32(np.inf)) if float(f) < v else f


def world_box(m, lo, hi):
    m = np.asarray(m, np.float32).astype(np.float64).reshape(3, 4)
    corners = np.array([[(hi if c & 1 else lo)[0], (hi if c & 2 else lo)[1], (hi if c & 4 else lo)[2]] for c in range(8)], np.float64)
    p = corners @ m[:, :3].T + m[:, 3]
    mn, mx = p.min(0), p.max(0)
    pad = PAD * max(np.abs(mn).max(), np.abs(mx).max())
    return np.array([_down(v - pad) for v in mn] + [_up(v + pad) for v in mx], np.float32)


def tree(boxes):
    """-> (records (k, 16) float32 with int bits in words 12-14, root box (6,), root ref) over world boxes (n, 6), n >= 1."""
    boxes = np.asarray(boxes, np.float32)
    recs = []

    def node(ids):
        if len(ids) == 1:
            return ~int(ids[0]), boxes[ids[0]]
        at = len(recs)
        recs.append(None)
        c = (boxes[ids, :3] + boxes[ids, 3:]) * np.float32(0.5)
        ext = c.max(0) - c.min(0)
        axis = 0
        if ext[1] > ext[axis]:
            axis = 1
        if ext[2] > ext[axis]:
            axis = 2
        order = sorted(range(len(ids)), key=lambda i: (float(c[i, axis]), int(ids[i])))
        s = [ids[i] for i in order]
        half = len(ids) // 2
        r0, b0 = node(s[:half])
        r1, b1 = node(s[half:])
        rec = np.zeros(16, np.float32)
        rec[0:6], rec[6:12] = b0, b1
        rec[12:15] = np.array([r0, r1, axis], np.int32).view(np.float32)
        recs[at] = rec
        return at, np.concatenate([np.minimum(b0[:3], b1[:3]), np.maximum(b0[3:], b1[3:])])

    ref, root = node(list(range(len(boxes))))
    return (np.array(recs, np.float32).reshape(-1, 16), root, ref)
