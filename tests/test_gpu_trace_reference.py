"""
GPU tests (-m gpu) of closest-hit and occlusion against the brute force of tests/trace_reference.py, which ignores the BVH, on the
designed scenes of tests/trace_cases.py and samples of the shipped ones, under every tree producer that applies: the upload, an
identity refit and a deforming refit (rt_update_triangles), rt_rebuild_bvh and rt_rebuild_bvh_ploc.

- The stepwise schedule with RT_OPT_TRAVERSAL 0 (trace_literal) and 1 (trace_fast on records in global memory): after
  rt_intersect(b) for every bounce up to 4, rt_read_rays(b) / rt_read_hits(b) of the two are byte-identical, equal the oracle
  tracing the device's tree (rt_read_bvh), and meet the brute-force rules (2 000 sampled rays per bounce), and the designed cases reach
  what they are built for at bounce 0 (trace_cases.REACH).
- The bodies that cannot be tapped per ray (staged records, octant records, RT_OPT_TOP_SMEM, PIN in k_frame, the shadow kernels):
  the one-kernel frame, the per-phase graph with octant records on and off, the fused steps and rt_integrate_samples give radiance
  bits and per-bounce counters (n_unoccluded included) equal to the stepwise context's and the oracle's, so the per-ray verdict
  carries over to them.
- The depth limits: a caller's tree of depth 65 and a PLOC tree of depth 65 are refused, and the refused PLOC rebuild changes
  nothing; the depth-64 chain, the depth-64 PLOC tree and the depth-43 LBVH are traced with a ray that defers depth - 1 entries.

The per-class counts of every case, producer and bounce are printed (pytest -s).
"""
import ctypes as C

import numpy as np
import pytest

from oracle.orcbind import Oracle
from raytracing_b200 import capi
from tests import trace_cases as T
from tests import trace_reference as R
from tests.helpers import bits
from tests.refit_model import deform
from tests.test_gpu_parity import check_stats, run_frame, schedule_ctx

pytestmark = pytest.mark.gpu

MB = 4
W, H = T.W, T.H
ALL = ("upload", "refit_identity", "refit_deform", "lbvh", "ploc")
PRODUCERS = {"chain64": ("upload", "refit_identity", "refit_deform"), "ploc64": ("upload", "ploc"), "lbvh_deep": ("upload", "lbvh"),
             "ties": ALL, "edges": ALL, "walls": ALL, "walls_axis": ALL,
             "CornellBox": ALL, "ShaderBalls": ("upload", "ploc"), "CornellBox_Dragon": ("upload", "lbvh")}
_cases = {}
_closest = {}


def closest(tris, rays):
    """The brute force of these rays, kept per (triangles, rays): it does not depend on the tree, and the producers of a case and
    the two traversals trace the same rays wherever their hits agree."""
    key = (R.digest(tris), R.digest(rays))
    if key not in _closest:
        _closest[key] = R.closest(tris, rays, t_min=0.0)
    return _closest[key]


def case(name):
    if name not in _cases:
        _cases[name] = T.case(name)
    return _cases[name]


def deformed(name, tris):
    return T.swap_axes(tris) if name.startswith("walls") else deform(tris, "noise", seed=5)


def produce(c, name, sc, producer):
    """Applies the producer to context c -> (the triangles it now holds, its tree as rt_read_bvh gives it)."""
    t = sc["triangles"]
    if producer == "refit_identity":
        c.update_triangles(t)
    elif producer == "refit_deform":
        t = deformed(name, t)
        c.update_triangles(t)
    elif producer in ("lbvh", "ploc"):
        c.rebuild_bvh("linear" if producer == "lbvh" else "ploc")
    return t, c.read_bvh()[0]


def depth(nodes):
    from tests.refit_model import levels
    return len(levels(nodes))


def zero_t_min(rays):
    r = rays.copy()
    r["origin"][:, 3] = 0.0            # the pixel word of the queue entry; the kernels trace from t = 0
    return r


def stepwise_bounces(name, producer):
    """Both traversals in lockstep on the stepwise schedule; -> (stepwise context (traversal 1), triangles, nodes)."""
    sc, cam = case(name)
    ctxs = [schedule_ctx("stepwise", sc, cam, W, H, ((capi.OPT_TRAVERSAL, m),)) for m in (0, 1)]
    try:
        for c in ctxs:
            tris, nodes = produce(c, name, sc, producer)
            c.reset(); c.generate_rays()
        orc = Oracle({**sc, "triangles": tris, "nodes": nodes})
        for b in range(MB + 1):
            got = []
            for c in ctxs:
                c.intersect(b)
                rays, pix = c.read_rays(b)
                hits, hpix = c.read_hits(b)
                assert np.array_equal(pix, hpix)
                order = np.argsort(pix, kind="stable")      # the queue order of later bounces is the shading pass's
                got.append((rays[order], pix[order], hits[order]))
            (rays, pix, hits), other = got[0], got[1]
            where = (name, producer, "bounce %d" % b)
            assert all(np.array_equal(x.view(np.uint8), y.view(np.uint8)) for x, y in zip((rays, pix, hits), other)), where
            if len(rays) == 0:
                break
            rays = zero_t_min(rays)
            oh, _ = orc.trace(rays)
            assert np.array_equal(oh.view(np.uint8), hits.view(np.uint8)), where
            pick = np.sort(np.random.default_rng(b).choice(len(rays), min(2000, len(rays)), replace=False))
            ref = closest(tris, rays[pick])
            rep = R.verdict(tris, rays[pick], nodes, hits["primitive_id"][pick], hits["bc"][pick], hits["t"][pick], where, t_min=0.0,
                            ref=ref, allow_box=0.0 if name in T.SHIPPED else 0.01)
            if b == 0 and name in T.REACH and producer != "refit_deform":
                got = T.reached(name, {**sc, "triangles": tris}, rays[pick], ref)
                assert all(got[k] >= v * len(pick) // (W * H) for k, v in T.REACH[name].items()), (where, got)
                rep.update(got)
            print(where, len(pick), rep)
            for c in ctxs:
                if b == 0:
                    c.compute_aovs()
                c.shade_miss(b); c.clear_outgoing_counter(b); c.clear_shadow_counter()
                c.shade_hits(b); c.intersect_shadow(); c.accumulate_direct()
        for c in ctxs:
            c.advance_sample_count()
        assert np.array_equal(bits(ctxs[0].read_radiance()), bits(ctxs[1].read_radiance())), (name, producer)
    except BaseException:
        ctxs[1].destroy()
        raise
    finally:
        ctxs[0].destroy()
    return ctxs[1], tris, nodes


RUNS = {"frame": ((capi.OPT_FRAME_KERNEL, 1),), "phase_graph": ((capi.OPT_FRAME_KERNEL, 0),),
        "phase_graph_canonical": ((capi.OPT_FRAME_KERNEL, 0), (capi.OPT_OCTANT_BVH, 0)),
        "phase_graph_global": ((capi.OPT_FRAME_KERNEL, 0), (capi.OPT_SMEM_BVH, 0)),
        "top_smem": ((capi.OPT_FRAME_KERNEL, 0), (capi.OPT_TOP_SMEM, 640)),
        "fused": ((capi.OPT_FRAME_KERNEL, 0),), "samples": ((capi.OPT_FRAME_KERNEL, 1),)}


def run(c, how):
    if how == "fused":
        c.generate_rays()
        for b in range(MB + 1):
            c.extend_shade(b); c.shadow_accumulate(b)
        c.advance_sample_count()
    elif how == "samples":
        c.integrate_samples(MB, 2)
    else:
        run_frame(c, how, MB)


@pytest.mark.parametrize("name", T.DESIGNED + T.SHIPPED)
def test_every_traversal_meets_the_brute_force(name):
    sc, cam = case(name)
    for producer in PRODUCERS[name]:
        step, tris, nodes = stepwise_bounces(name, producer)
        try:
            want, want_st = bits(step.read_radiance()), step.frame_stats()
            orc = Oracle({**sc, "triangles": tris, "nodes": nodes})
            orad, _, ost = orc.render(cam, W, H, MB)
            orad2 = bits(orc.render(cam, W, H, MB, sample_idx=1, radiance=orad.copy())[0][..., :3])
            assert np.array_equal(want[..., :3], bits(orad[..., :3])), (name, producer, "stepwise")
            check_stats(want_st, ost, MB, (name, producer, "stepwise"))
            runs = [r for r in RUNS if r != "top_smem" or name in ("lbvh_deep", "ShaderBalls")]
            for how in runs:
                c = schedule_ctx(None, sc, cam, W, H, RUNS[how])
                try:
                    produce(c, name, sc, producer)
                    c.reset(); run(c, how)
                    where = (name, producer, how)
                    if how == "samples":              # two samples in one call: the oracle's samples 0 and 1
                        assert np.array_equal(bits(c.read_radiance()[..., :3]), orad2), where
                        continue
                    assert np.array_equal(bits(c.read_radiance()), want), where
                    check_stats(c.frame_stats(), ost, MB, where)
                finally:
                    c.destroy()
        finally:
            step.destroy()


@pytest.mark.parametrize("name", ["chain64", "ploc64", "lbvh_deep"])
def test_deep_trees_defer_depth_minus_one_entries(name):
    """The device's tree has the stated depth (64, 64, >= 40 and <= 62), and the camera ray that defers the most entries under the
    literal rule holds depth - 1 of them; the oracle visits the nodes the stack model visits, and the device's hit on that ray is
    the brute-force closest."""
    sc, cam = case(name)
    producer = {"chain64": "upload", "ploc64": "ploc", "lbvh_deep": "lbvh"}[name]
    c = schedule_ctx("stepwise", sc, cam, W, H)
    try:
        tris, nodes = produce(c, name, sc, producer)
        dep = depth(nodes)
        assert dep == 64 if name != "lbvh_deep" else 40 <= dep <= 62, (name, dep)
        c.reset(); c.generate_rays(); c.intersect(0)
        rays, _ = c.read_rays(0)
        hits, _ = c.read_hits(0)
    finally:
        c.destroy()
    rays = zero_t_min(rays)
    deferred = [T.deferred_entries(nodes, rays["origin"][k, :3], rays["direction"][k, :3]) for k in range(len(rays))]
    k = int(np.argmax([dfr for dfr, _ in deferred]))
    assert deferred[k][0] == dep - 1, (name, deferred[k], dep)
    _, counters = Oracle({**sc, "triangles": tris, "nodes": nodes}).trace(rays[k: k + 1])
    assert counters[0] == deferred[k][1], (name, counters, deferred[k])
    R.verdict(tris, rays[k: k + 1], nodes, hits["primitive_id"][k: k + 1], hits["bc"][k: k + 1], hits["t"][k: k + 1], (name, k),
              t_min=0.0, allow_box=0.0)
    print(name, "depth", dep, "deferred", deferred[k][0], "ray", k)


def test_depth_65_is_refused():
    """A caller's tree of depth 65 is refused by the upload; a PLOC tree of depth 65 gives RT_ERR_UNSUPPORTED and leaves the tree
    and the frames as they were."""
    sc65 = T.chain(64)
    c = capi.Context(W, H)
    try:
        with pytest.raises(capi.RtError) as e:
            c.upload_scene(sc65)
        assert e.value.code == -1 and "deeper" in str(e.value)
    finally:
        c.destroy()
    sc = T.geometric_chain(65)
    cam = T.chain_camera()
    c = schedule_ctx(None, sc, cam, W, H)
    try:
        c.reset(); c.integrate(MB)
        want = bits(c.read_radiance())
        nodes, rec = c.read_bvh()
        n = C.c_uint64(7)
        assert c.lib.rt_rebuild_bvh_ploc(c.h, C.byref(n)) == -5 and n.value == 7
        nodes2, rec2 = c.read_bvh()
        assert np.array_equal(nodes.view(np.uint8), nodes2.view(np.uint8)) and np.array_equal(bits(rec), bits(rec2))
        c.reset(); c.integrate(MB)
        assert np.array_equal(bits(c.read_radiance()), want)
    finally:
        c.destroy()
