"""
GPU tests (-m gpu) of the two-level traversal of instanced scenes against the brute force of tests/instance_reference.py, which
ignores the top-level tree, the world boxes and the meshes' trees, on the cases of test_instance_trace_reference_cpu.py.

- Per ray, on the stepwise schedule: after rt_intersect(b) for every bounce up to 4, rt_read_rays(b) / rt_read_hits(b) sorted by
  pixel equal the CPU model's traversal of the same rays (InstanceModel.trace_instanced) byte for byte, and 2 000 sampled rays per
  bounce meet the brute force's rules (a lost hit only where the mesh's own tree loses it too).
- The schedules that cannot be tapped per ray (the default graph, overlap 0 / 1, PDL off, the one-kernel frame, the fused steps and
  rt_integrate_samples): radiance bits and per-bounce counters (n_unoccluded included) equal the stepwise context's and the model's
  frame, so the per-ray verdict carries over to them, the device's shadow rays included.
- How the instances and meshes got there: rt_set_instances straight after the upload; a second rt_set_instances after a different
  list; rt_update_mesh_triangles with noise; and a move that takes the mesh outside its old root box, so that the world boxes must
  follow the update.

The per-class counts of every case, history and bounce are printed (pytest -s).
"""
import numpy as np
import pytest

from raytracing_b200 import capi
from tests.helpers import bits
from tests.instance_model import InstanceModel
from tests import instance_reference as IR
from tests.refit_model import deform, refit
from tests.test_gpu_instancing import STAT_KEYS, inst_ctx
from tests.test_gpu_parity import run_frame
from tests.test_instance_trace_reference_cpu import ALLOW_MESH_LOST, CASES

pytestmark = pytest.mark.gpu

MB = 4
W, H = 96, 64
NAMES = ("placements_CornellBox", "far_ill_conditioned", "far_ill_conditioned_small", "coinciding", "single_leaf", "offset_mesh")
HISTORIES = ("upload", "relist", "mesh_noise", "mesh_moved")
RUNS = {"default": (), "overlap0": ((capi.OPT_OVERLAP, 0),), "overlap1": ((capi.OPT_OVERLAP, 1),), "no_pdl": ((capi.OPT_PDL, 0),),
        "frame_kernel": ((capi.OPT_FRAME_KERNEL, 1),), "fused": ((capi.OPT_FRAME_KERNEL, 0),), "samples": ()}


def moved_tris(tris, nodes):
    """The mesh moved by 1.5 of its extent along x: outside its old root box."""
    t = tris.copy()
    ext = float((nodes["bounds_max"][0, :3] - nodes["bounds_min"][0, :3]).max())
    for v in ("v1", "v2", "v3"):
        t[v]["position"][:, 0] += np.float32(1.5 * ext)
    return t


def history_ctx(name, history, options=()):
    """-> (context, meshes as a fresh upload would take them, shared, ids, mats, camera) after the history."""
    meshes, shared, ids, mats, cam = CASES[name]()
    if history == "relist":
        other = mats[::-1].copy()
        other[:, :, 3] += np.float32(0.25)
        c = inst_ctx(meshes, shared, [ids[-1]] * len(other) if len(ids) else [], other, w=W, h=H, cam=cam, options=options)
        c.set_instances(ids, mats)
    else:
        c = inst_ctx(meshes, shared, ids, mats, w=W, h=H, cam=cam, options=options)
    if history in ("mesh_noise", "mesh_moved"):
        m = meshes[0]
        t = deform(m["triangles"], "noise", seed=5) if history == "mesh_noise" else moved_tris(m["triangles"], m["nodes"])
        c.update_mesh_triangles(0, t)
        meshes = [{"triangles": t, "nodes": refit(m["nodes"], t)}] + list(meshes[1:])
    return c, meshes, shared, ids, mats, cam


def stepwise(name, history):
    """Per-ray checks on the stepwise schedule; -> (stepwise context, meshes, shared, ids, mats, camera)."""
    c, meshes, shared, ids, mats, cam = history_ctx(name, history)
    try:
        model = InstanceModel(meshes, shared)
        ref_scene = IR.Scene(meshes, ids, mats)
        c.reset(); c.generate_rays()
        for b in range(MB + 1):
            c.intersect(b)
            rays, pix = c.read_rays(b)
            hits, hpix = c.read_hits(b)
            assert np.array_equal(pix, hpix)
            order = np.argsort(pix, kind="stable")
            rays, hits = rays[order], hits[order]
            where = (name, history, "bounce %d" % b)
            if len(rays) == 0:
                break
            rays = rays.copy()
            rays["origin"][:, 3] = 0.0              # the pixel word of the queue entry; the kernels trace from t = 0
            want = model.trace_instanced(ids, mats, rays)
            assert np.array_equal(want.view(np.uint8), hits.view(np.uint8)), where
            pick = np.sort(np.random.default_rng(b).choice(len(rays), min(2000, len(rays)), replace=False))
            r = rays[pick]
            ref = ref_scene.closest(r)
            got_t = np.where(hits["primitive_id"][pick] != 0xFFFFFFFF, hits["t"][pick], np.float32(np.inf))
            lost = ref_scene.mesh_lost(model, r, got_t, ref)
            rep = ref_scene.verdict(r, hits["primitive_id"][pick], hits["bc"][pick], hits["t"][pick], where, ref=ref,
                                    allow_box=ALLOW_MESH_LOST, lost=lost)
            print(where, len(pick), rep)
            if b == 0:
                c.compute_aovs()
            c.shade_miss(b); c.clear_outgoing_counter(b); c.clear_shadow_counter()
            c.shade_hits(b); c.intersect_shadow(); c.accumulate_direct()
        c.advance_sample_count()
    except BaseException:
        c.destroy()
        raise
    return c, meshes, shared, ids, mats, cam


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


@pytest.mark.parametrize("history", HISTORIES)
@pytest.mark.parametrize("name", NAMES)
def test_instanced_traversal_meets_the_brute_force(name, history):
    step, meshes, shared, ids, mats, cam = stepwise(name, history)
    try:
        want = bits(step.read_radiance()[..., :3])
        st = step.frame_stats()
        model = InstanceModel(meshes, shared)
        mrad, _, mst, _ = model.render_instanced(ids, mats, cam, W, H, MB)
        assert np.array_equal(want, bits(mrad[..., :3])), (name, history, "stepwise")
        for k in STAT_KEYS:
            assert np.array_equal(st[k][: MB + 1], mst[k][: MB + 1]), (name, history, "stepwise", k)
        mrad2 = bits(model.render_instanced(ids, mats, cam, W, H, MB, sample_idx=1, radiance=mrad.copy())[0][..., :3])
    finally:
        step.destroy()
    for how, opts in RUNS.items():
        c, *_ = history_ctx(name, history, options=opts)
        try:
            c.reset()
            run(c, how)
            where = (name, history, how)
            got = bits(c.read_radiance()[..., :3])
            if how == "samples":                    # two samples in one call: the model's samples 0 and 1
                assert np.array_equal(got, mrad2), where
                continue
            assert np.array_equal(got, want), where
            gst = c.frame_stats()
            for k in STAT_KEYS:
                assert np.array_equal(gst[k][: MB + 1], mst[k][: MB + 1]), (where, k)
        finally:
            c.destroy()
