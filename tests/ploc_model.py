"""
Independent numpy statement of the build rule of rt_rebuild_bvh_ploc (include/rt_b200.h): parallel locally-ordered clustering
(Meister & Bittner 2018) over the triangles in the key order of rt_rebuild_bvh, one triangle per leaf.  Each iteration finds every
cluster's nearest neighbour within RADIUS positions (every pair's distance computed once, ties broken by one key per pair rather
than per candidate as the kernel does), merges the mutual pairs and compacts the list; the tree is then numbered in
preorder from the subtree sizes, level by level, the records breadth-first for the top and depth-first for the rest, and the
boxes come from tests/refit_model.refit.  Vectorised per iteration, so it runs on Synthetic10M.
"""
import numpy as np

from raytracing_b200.layouts import NODE_DT
from tests.lbvh_model import LEAF, TOP_RECORDS, sorted_keys
from tests.refit_model import FLT_MAX, refit, vmax, vmin

RADIUS = 16
MAX_DEPTH = 64


def area(lo, hi):
    """A(lo, hi) = (ex*ey + ey*ez) + ez*ex with e = hi - lo, float32; +inf unless >= 0 and finite."""
    with np.errstate(invalid="ignore", over="ignore"):
        e = hi - lo
        a = (e[:, 0] * e[:, 1] + e[:, 1] * e[:, 2]) + e[:, 2] * e[:, 0]
        return np.where((a >= 0) & np.isfinite(a), a, np.float32(np.inf))


def leaf_boxes(triangles):
    """The refit rule's box of each triangle as a one-triangle leaf: (lo, hi), (n, 3) float32 each."""
    p = [np.ascontiguousarray(triangles[v]["position"][:, :3], dtype=np.float32) for v in ("v1", "v2", "v3")]
    lo = vmin(np.float32(FLT_MAX), vmin(vmin(p[0], p[1]), p[2]))
    hi = vmax(np.float32(-FLT_MAX), vmax(vmax(p[0], p[1]), p[2]))
    return lo.astype(np.float32), hi.astype(np.float32)


def tie_key(i, j):
    """The order of pairs (i < j) at equal distance: the smaller gap j - i, then an even i, then the smaller i."""
    return (((j - i) * 2 + (i & 1)) << 40) + i


def cluster(triangles, radius=RADIUS):
    """The clustering of steps 1-5 -> (children int64 (n - 1, 2) of interior node k as node references (a leaf is its triangle
    id, interior node k is n + k, k in creation order), axis uint32 (n - 1), leaves int64 (n - 1) under interior node k, root
    reference, iterations, keys)."""
    n = len(triangles)
    keys = sorted_keys(triangles)
    ids = (keys & np.uint64(0xFFFFFFFF)).astype(np.int64)
    blo, bhi = leaf_boxes(triangles)
    lo, hi, ref, cnt = blo[ids], bhi[ids], ids.copy(), np.ones(n, np.int64)
    children = np.zeros((max(n - 1, 0), 2), np.int64)
    axis = np.zeros(max(n - 1, 0), np.uint32)
    leaves = np.zeros(max(n - 1, 0), np.int64)
    made, iterations = 0, 0
    while len(ref) > 1:
        c = len(ref)
        pos = np.arange(c)
        best_d = np.full(c, np.inf, np.float32)
        best_t = np.full(c, np.iinfo(np.int64).max, np.int64)
        best_j = np.full(c, -1, np.int64)
        for o in range(1, radius + 1):
            i = pos[: max(c - o, 0)]
            j = i + o
            d = area(vmin(lo[i], lo[j]), vmax(hi[i], hi[j]))         # Union with the lower position first
            tie = tie_key(i, j)
            for me, other in ((i, j), (j, i)):
                take = (d < best_d[me]) | ((d == best_d[me]) & (tie < best_t[me]))
                best_d[me[take]], best_t[me[take]], best_j[me[take]] = d[take], tie[take], other[take]
        nn = best_j
        mutual = nn[nn] == pos
        low = np.flatnonzero(mutual & (pos < nn))
        assert low.size > 0, "an iteration without a merge"
        high = nn[low]
        cl, ch = lo[low] + hi[low], lo[high] + hi[high]
        dl = np.abs(ch - cl)
        r = np.arange(low.size)
        ax = np.zeros(low.size, np.int64)
        ax = np.where(dl[:, 1] > dl[r, ax], 1, ax)
        ax = np.where(dl[:, 2] > dl[r, ax], 2, ax)
        h_first = ch[r, ax] < cl[r, ax]
        k = made + r
        children[k, 0] = np.where(h_first, ref[high], ref[low])
        children[k, 1] = np.where(h_first, ref[low], ref[high])
        axis[k] = ax
        leaves[k] = cnt[low] + cnt[high]
        lo[low], hi[low] = vmin(lo[low], lo[high]), vmax(hi[low], hi[high])
        ref[low], cnt[low] = n + k, leaves[k]
        made += low.size
        keep = ~(mutual & (pos > nn))
        lo, hi, ref, cnt = lo[keep], hi[keep], ref[keep], cnt[keep]
        iterations += 1
    assert made == n - 1
    return children, axis, leaves, int(ref[0]), iterations, keys


def build(triangles, with_boxes=True, radius=RADIUS):
    """-> (nodes NODE_DT[2n - 1] in the rule's preorder layout with refit boxes, info dict: keys, iterations, max_depth (levels,
    root = 1), depth_error (max_depth > 64: the call returns RT_ERR_UNSUPPORTED), top_n, record of each interior node in
    preorder, bfs)."""
    n = len(triangles)
    children, axis, leaves, root, iterations, keys = cluster(triangles, radius)
    nodes = np.zeros(2 * n - 1, dtype=NODE_DT)
    size = np.concatenate([np.ones(n, np.int64), leaves])                # leaves under each node reference
    cur, pre = np.array([root], np.int64), np.array([0], np.int64)
    depth, bfs_interior = 0, []
    while cur.size:
        depth += 1
        leaf = cur < n
        nodes["offset"][pre[leaf]] = cur[leaf]
        nodes["num_primitives_axis"][pre[leaf]] = LEAF
        k, ip = cur[~leaf] - n, pre[~leaf]
        if not k.size:
            break
        bfs_interior.append(ip)
        right = ip + 2 * size[children[k, 0]]
        nodes["offset"][ip] = right
        nodes["num_primitives_axis"][ip] = axis[k]
        cur = children[k].ravel()
        pre = np.stack([ip + 1, right], 1).ravel()
    info = {"keys": keys, "iterations": iterations, "max_depth": depth, "depth_error": depth > MAX_DEPTH}
    bfs = np.concatenate(bfs_interior) if bfs_interior else np.zeros(0, np.int64)
    top_n = min(n - 1, TOP_RECORDS)
    record = np.full(2 * n - 1, -1, np.int64)
    record[bfs[:top_n]] = np.arange(top_n)
    rest = np.sort(bfs[top_n:])                                          # depth-first = preorder
    record[rest] = top_n + np.arange(rest.size)
    info.update(top_n=top_n, record=record, bfs=bfs)
    return (refit(nodes, triangles) if with_boxes else nodes), info


def sah_cost(nodes):
    """SAH cost with C_node = C_tri = 1 on the nodes' boxes, each area relative to the root's."""
    a = area(nodes["bounds_min"][:, :3].astype(np.float64), nodes["bounds_max"][:, :3].astype(np.float64))
    count = (nodes["num_primitives_axis"] >> 16).astype(np.float64)
    w = np.where(count > 0, count, 1.0)
    return float((a * w).sum() / a[0])
