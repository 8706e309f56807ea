"""
Independent numpy statement of the build rule of rt_rebuild_bvh (include/rt_b200.h): a linear BVH over the current triangles.
Sorts with numpy, builds the topology top-down one level at a time by splitting sorted key ranges where their highest
differing bit flips (a binary search per range, not the Karras construction the kernels use), numbers the nodes in preorder
from the subtree sizes, the records breadth-first for the top and depth-first for the rest, and takes the boxes from
tests/refit_model.refit.  Vectorised per tree level, so it runs on Synthetic10M.
"""
import numpy as np

from raytracing_b200.layouts import NODE_DT
from tests.refit_model import refit

TOP_RECORDS = 1024
LEAF = 1 << 16


def key_points(triangles):
    """s = (p1 + p2) + p3 per component, float32: (n, 3)."""
    p = [np.ascontiguousarray(triangles[v]["position"][:, :3], dtype=np.float32) for v in ("v1", "v2", "v3")]
    return (p[0] + p[1]) + p[2]


def quantize(s):
    """10-bit cell per axis: (n, 3) uint32."""
    q = np.zeros(s.shape, np.uint32)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        for a in range(3):
            x = s[:, a]
            fin = np.isfinite(x)
            if not fin.any():
                continue
            lo, hi = x[fin].min(), x[fin].max()
            k = np.float32(1024.0) / (hi - lo) if hi > lo else np.float32(0.0)
            v = (x - lo) * np.float32(k)
            qa = np.where(v >= np.float32(1023.0), np.uint32(1023), np.where(v > 0, np.trunc(np.where(v > 0, v, 0)), 0)).astype(np.uint32)
            q[:, a] = np.where(fin, qa, np.uint32(0))
    return q


def morton(q):
    """Bit j of qx -> bit 3j+2, qy -> 3j+1, qz -> 3j (30 bits)."""
    code = np.zeros(q.shape[0], np.uint64)
    for j in range(10):
        for a, sh in ((0, 2), (1, 1), (2, 0)):
            code |= ((q[:, a].astype(np.uint64) >> np.uint64(j)) & np.uint64(1)) << np.uint64(3 * j + sh)
    return code


def sorted_keys(triangles):
    n = len(triangles)
    code = morton(quantize(key_points(triangles)))
    keys = (code << np.uint64(32)) | np.arange(n, dtype=np.uint64)
    return np.sort(keys)


def highest_bit(x):
    """Index of the highest set bit of each (non-zero) uint64."""
    h = np.zeros(x.shape, np.int64)
    v = x.copy()
    for s in (32, 16, 8, 4, 2, 1):
        m = v >= (np.uint64(1) << np.uint64(s))
        h[m] += s
        v[m] >>= np.uint64(s)
    return h


def build(triangles, with_boxes=True):
    """-> (nodes NODE_DT[2n - 1] in the rule's preorder layout with refit boxes, info dict: keys, max_depth (levels of the
    build_layout walk, root = 1), top_n, record of each interior node in preorder)."""
    n = len(triangles)
    keys = sorted_keys(triangles)
    ids = (keys & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    nodes = np.zeros(2 * n - 1, dtype=NODE_DT)
    if n == 1:
        nodes[0]["offset"] = ids[0]; nodes[0]["num_primitives_axis"] = LEAF
        return (refit(nodes, triangles) if with_boxes else nodes), {"keys": keys, "max_depth": 1, "top_n": 0, "bfs": np.zeros(0, np.int64)}
    # level by level: ranges [a, b] with their preorder index; interior ranges split, leaves are written
    a = np.array([0], np.int64); b = np.array([n - 1], np.int64); pre = np.array([0], np.int64)
    depth = 0
    bfs_interior = []                    # preorder indices of interior nodes, breadth-first (children first / second)
    while a.size:
        depth += 1
        leaf = a == b
        lp, la = pre[leaf], a[leaf]
        nodes["offset"][lp] = ids[la]
        nodes["num_primitives_axis"][lp] = LEAF
        ia, ib, ip = a[~leaf], b[~leaf], pre[~leaf]
        if not ia.size:
            break
        bfs_interior.append(ip)
        h = highest_bit(keys[ia] ^ keys[ib])
        thresh = ((keys[ia] >> h.astype(np.uint64)) + np.uint64(1)) << h.astype(np.uint64)
        g = np.searchsorted(keys, thresh, side="left") - 1             # the last key of the first child
        assert ((g >= ia) & (g < ib)).all()
        axis = np.where(h >= 32, 2 - ((h - 32) % 3), 0)
        right = ip + 2 * (g - ia + 1)
        nodes["offset"][ip] = right
        nodes["num_primitives_axis"][ip] = axis
        # next level, children interleaved (first, second) per parent in this level's order
        a = np.stack([ia, g + 1], 1).ravel(); b = np.stack([g, ib], 1).ravel(); pre = np.stack([ip + 1, right], 1).ravel()
    bfs = np.concatenate(bfs_interior)
    top_n = min(n - 1, TOP_RECORDS)
    record = np.full(2 * n - 1, -1, np.int64)
    record[bfs[:top_n]] = np.arange(top_n)
    rest = np.sort(bfs[top_n:])                                          # depth-first = preorder
    record[rest] = top_n + np.arange(rest.size)
    info = {"keys": keys, "max_depth": depth, "top_n": top_n, "record": record, "bfs": bfs}
    return (refit(nodes, triangles) if with_boxes else nodes), info
