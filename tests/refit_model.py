"""
Independent numpy statement of the BVH refit rule of rt_update_triangles (include/rt_b200.h), vectorised level by level:
min(a, b) = (b < a) ? b : a and max(a, b) = (a < b) ? b : a per component (std::min / std::max as the reference's Bounds3 uses
them); a leaf folds Union(Bounds3(p1, p2), p3) of its triangles in leaf order into (FLT_MAX, -FLT_MAX); an interior box is
Union(first child, second child).  Only the xyz of the boxes of nodes reachable from the root change.
"""
import numpy as np

FLT_MAX = np.float32(np.finfo(np.float32).max)


def vmin(a, b):
    return np.where(b < a, b, a)


def vmax(a, b):
    return np.where(a < b, b, a)


def levels(nodes):
    """Reachable node indices, one array per depth (root first)."""
    count = nodes["num_primitives_axis"] >> 16
    out, cur = [], np.array([0], dtype=np.int64)
    while cur.size:
        out.append(cur)
        inner = cur[count[cur] == 0]
        cur = np.concatenate([inner + 1, nodes["offset"][inner].astype(np.int64)])
    return out


def refit(nodes, triangles):
    """The node array after a refit of `nodes` (an uploaded tree) over `triangles` (leaf order)."""
    out = nodes.copy()
    count = (nodes["num_primitives_axis"] >> 16).astype(np.int64)
    off = nodes["offset"].astype(np.int64)
    p = [np.ascontiguousarray(triangles[v]["position"][:, :3], dtype=np.float32) for v in ("v1", "v2", "v3")]
    lo = np.zeros((len(nodes), 3), np.float32)
    hi = np.zeros((len(nodes), 3), np.float32)
    lv = levels(nodes)
    leaves = np.concatenate([l[count[l] > 0] for l in lv])
    blo = np.full((leaves.size, 3), FLT_MAX, np.float32)
    bhi = np.full((leaves.size, 3), -FLT_MAX, np.float32)
    for k in range(int(count[leaves].max())):
        sel = count[leaves] > k
        t = off[leaves[sel]] + k
        tlo = vmin(vmin(p[0][t], p[1][t]), p[2][t])
        thi = vmax(vmax(p[0][t], p[1][t]), p[2][t])
        blo[sel] = vmin(blo[sel], tlo)
        bhi[sel] = vmax(bhi[sel], thi)
    lo[leaves], hi[leaves] = blo, bhi
    for l in reversed(lv):
        inner = l[count[l] == 0]
        a, b = inner + 1, off[inner]
        lo[inner] = vmin(lo[a], lo[b])
        hi[inner] = vmax(hi[a], hi[b])
    reach = np.concatenate(lv)
    out["bounds_min"][reach, :3] = lo[reach]
    out["bounds_max"][reach, :3] = hi[reach]
    return out


def records_match_nodes(nodes, records):
    """Every traversal record's two child boxes equal its children's node boxes (bits), found by walking both layouts from
    the root (record 0); returns the number of records checked."""
    rec_i = records.view("<i4")
    count = nodes["num_primitives_axis"] >> 16
    if count[0] > 0:
        return 0
    stack, seen = [(0, 0)], 0
    while stack:
        node, r = stack.pop()
        seen += 1
        kids = (node + 1, int(nodes["offset"][node]))
        for s, child in enumerate(kids):
            box = records[r, 6 * s: 6 * s + 6]
            want = np.concatenate([nodes["bounds_min"][child, :3], nodes["bounds_max"][child, :3]])
            assert np.array_equal(box.view("<u4"), want.view("<u4")), (node, s, box, want)
            ref = int(rec_i[r, 12 + s])
            if count[child] == 0:
                stack.append((child, ref))
            else:
                assert ref == ~int(nodes["offset"][child]), (node, s, ref)
    return seen


def deform(triangles, kind, seed=1, amount=0.05):
    """Seeded deformations of a leaf-ordered triangle array: 'noise' moves every vertex (shared vertices apart), 'rigid' moves a
    random subset of triangles by one offset, 'scale' scales the scene about the origin."""
    rng = np.random.default_rng(seed)
    t = triangles.copy()
    pos = np.stack([t[v]["position"][:, :3] for v in ("v1", "v2", "v3")], axis=1)      # (n, 3, 3)
    ext = np.float32(np.ptp(pos.reshape(-1, 3), axis=0).max())
    if kind == "noise":
        pos = pos + (rng.standard_normal(pos.shape) * amount * 0.1 * ext).astype(np.float32)
    elif kind == "rigid":
        sel = rng.random(len(t)) < 0.3
        pos[sel] = pos[sel] + (rng.standard_normal(3) * amount * ext).astype(np.float32)
    elif kind == "scale":
        pos = pos * np.float32(1.0 + amount)
    else:
        raise ValueError(kind)
    pos = pos.astype(np.float32)
    for i, v in enumerate(("v1", "v2", "v3")):
        t[v]["position"][:, :3] = pos[:, i]
    return t
