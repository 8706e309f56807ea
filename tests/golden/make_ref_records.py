#!/usr/bin/env python3
"""
tests/golden/make_ref_records.py — what the REFERENCE's own code (oracle/_ref/libref.so and libref_libm.so, built by
oracle/build_ref.py from the reference tree) produces for the cases of tests/test_oracle_vs_ref.py and of the reference
comparisons in tests/test_host.py, stored so that those tests run without the reference.

    python tests/golden/make_ref_records.py [--reference <reference tree>]

Writes into tests/golden/ref/:
  frames.json.xz    per case and sample: per-bounce counters and the sha256 digests of the radiance bits and primary hits
                    (tests/helpers.frame_record);
  libm_sample.npz   a seeded sample of the pixels of the libm build's frames (test_math_library_sensitivity_is_small);
  loader.json.xz    digests of the scene arrays / texels the reference's Scene loader made of generated OBJ, HDR and image files;
and tests/golden/scenes/input_order.npz.xz: per shipped scene, the triangle order (offsets from the order of the stored dump) in
which tests/test_host.py::shipped_scene_inputs writes its OBJ so that the reference's own loader and Bvh::BuildCPU rebuild
exactly the stored arrays; the reference's LoadHDR is checked to read the re-encoded environment back bit for bit.
"""
import argparse
import json
import lzma
import os
import pathlib
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, REPO)

from oracle import refbind  # noqa: E402
from raytracing_b200.camera import default_camera  # noqa: E402
from tests import test_host as H  # noqa: E402
from tests import test_oracle_vs_ref as T  # noqa: E402
from tests.helpers import bits, digest, frame_record, fuzz_configs, scene, synthetic_sampler_tables  # noqa: E402


def ref_samples(sc, cam, w, h, mb, n, wf=False, with_hits=True, keys=None, tables=None, keep=None):
    """Records of n accumulated samples of the reference's Integrate(), or of the samples (0-based) listed in `keep`."""
    r = refbind.RefRenderer().open_arrays(sc)
    r.begin(w, h); r.set_camera(cam); r.set_max_bounces(mb); r.enable_white_furnace(wf)
    if tables is not None:
        r.use_sampler_tables(tables); r.set_blue_noise(True)
    out = []
    for sample in range(n):
        r.integrate()
        if keep is not None and sample not in keep:
            continue
        kw = {"keys": keys} if keys else {}
        out.append(frame_record(r.stats(), mb, r.radiance(), r.primary_hits() if with_hits else None, **kw))
    r.close()
    return out


def oracle_vs_ref_frames():
    F = {}
    for name, w, h, mb, wf in T.BIT_EXACT_CASES:
        F["bit_exact/%s_%dx%d_b%d_wf%d" % (name, w, h, mb, wf)] = ref_samples(scene(name), default_camera(w, h), w, h, mb, 2, wf)
    for name in T.AOV_CASES:
        w, h, mb = 128, 72, 3
        r = refbind.RefRenderer().open_arrays(scene(name)); r.begin(w, h)
        r.enable_denoiser(True); r.set_max_bounces(mb)
        recs = []
        for cam in T.aov_cameras(w, h):
            r.set_camera(cam); r.integrate()
            recs.append({"albedo": digest(bits(r.aov_albedo()[..., :3])), "depth": digest(bits(r.aov_depth())),
                         "normal": digest(bits(r.aov_normal()[..., :3])), "velocity": digest(bits(r.aov_velocity())),
                         "radiance": digest(bits(r.radiance()[..., :3])), "resolved": digest(bits(r.resolved()))})
        r.close()
        F["aov/" + name] = recs
    from tests.scenes_extra import many_lights_scene, textured_cornell
    F["textured"] = ref_samples(textured_cornell(), default_camera(96, 64), 96, 64, 4, 1, with_hits=False,
                                keys=("n_ext", "n_miss", "n_shadow", "n_cont", "n_unoccluded"))
    for name, w, h, mb, wf in T.BLUE_NOISE_CASES:
        F["blue_noise/%s_%dx%d_b%d_wf%d" % (name, w, h, mb, wf)] = ref_samples(scene(name), default_camera(w, h), w, h, mb, 3, wf,
                                                                              with_hits=False, tables=synthetic_sampler_tables())
    for name, w, h, mb in T.LIGHTS_CASES:
        F["lights/%s_%dx%d_b%d" % (name, w, h, mb)] = ref_samples(many_lights_scene(name), T.lights_camera(w, h), w, h, mb, 2)
    for case, (name, w, h, mb, kw) in T.DEGENERATE_CASES.items():
        F["degenerate/" + case] = ref_samples(scene(name), default_camera(w, h, **kw), w, h, mb, 2)
    for i, (name, w, h, mb, kw, wf) in enumerate(fuzz_configs()):
        F["fuzzed/%d" % i] = ref_samples(scene(name), default_camera(w, h, **kw), w, h, mb, 2, wf)
    from tests.scenes_extra import closed_cornell
    for w, h, mb, sampler in T.LONG_PATH_CASES:
        F["long_path/closed_cornell_%dx%d_b%d_%s" % (w, h, mb, sampler)] = ref_samples(closed_cornell(), default_camera(w, h), w, h, mb, 2,
                                                                                      tables=T.sampler_tables(sampler))
    for name, w, h, mb, sampler in T.LATE_SAMPLE_CASES:
        F["late_sample/%s_%dx%d_b%d_%s" % (name, w, h, mb, sampler)] = ref_samples(scene(name), default_camera(w, h), w, h, mb,
                                                                                  T.LATE_SAMPLE_COUNT, tables=T.sampler_tables(sampler),
                                                                                  keep=T.LATE_SAMPLE_KEEP)
    return F


def generated_obj_frames(reference):
    F = {}
    for seed in H.GENERATED_OBJ_SEEDS:
        with tempfile.TemporaryDirectory() as tmp:
            obj, cam, w, h, mb = H.generated_obj_case(tmp, seed)
            r = refbind.RefRenderer().open_obj(reference, obj)
            r.begin(w, h); r.set_camera(cam); r.set_max_bounces(mb); r.integrate()
            F["generated_obj/%d" % seed] = [frame_record(r.stats(), mb, r.radiance(), r.primary_hits(), keys=("n_ext",))]
            r.close()
    return F


def libm_samples():
    out = {}
    for name, w, h, mb, _ in T.LIBM_CASES:
        r = refbind.RefRenderer(libm=True).open_arrays(scene(name))
        r.begin(w, h); r.set_camera(default_camera(w, h)); r.set_max_bounces(mb); r.integrate()
        out[name] = r.radiance()[..., :3].reshape(-1, 3)[T.libm_sample_index(w, h)].astype("<f4")
        r.close()
    return out


def shipped_scene_orders(reference):
    """Input order of each shipped scene's triangles for which the reference rebuilds the stored tree and leaf order: start from
    the stored (leaf) order and move every triangle to where the reference's builder put it, until the output is the stored order."""
    from tests.golden.make_obj_fixtures import reference_env
    out = {}
    for name in H.SHIPPED_SCENES:
        g = scene(name)
        n = len(g["triangles"])
        def key(t):                  # what the test compares of a triangle (the padding words are not initialised)
            cols = [t[v][f][:, :k] for v in ("v1", "v2", "v3") for f, k in (("position", 3), ("normal", 3), ("texcoord", 2))]
            return [r.tobytes() for r in np.ascontiguousarray(np.concatenate(cols + [t["mtlIndex"][:, None].view("<f4")], 1))]
        slot = {k: i for i, k in enumerate(key(g["triangles"]))}
        order = np.arange(n)
        with tempfile.TemporaryDirectory() as tmp:
            for _ in range(8):
                obj, hdr = H.shipped_scene_inputs(tmp, name, order)
                r = refbind.RefRenderer().open_obj(reference, obj)
                got = r.scene(); r.close()
                landed = np.array([slot[k] for k in key(got["triangles"])])     # stored index of the triangle in each output slot
                if (landed == np.arange(n)).all():
                    break
                where = np.empty(n, dtype=np.int64); where[landed] = np.arange(n)
                order = where[order]
            else:
                raise SystemExit(name + ": no input order reproduces the stored leaf order")
            for k in ("bounds_min", "bounds_max"):
                assert np.array_equal(bits(got["nodes"][k][:, :3]), bits(g["nodes"][k][:, :3])), (name, k)
            for k in ("offset", "num_primitives_axis"):
                assert np.array_equal(got["nodes"][k], g["nodes"][k]), (name, k)
            for k in ("materials", "emissive", "scene_info"):
                assert got[k].tobytes() == g[k].tobytes(), (name, k)
            with open(hdr, "rb") as f:
                root = os.path.join(tmp, "env"); os.makedirs(root)
                env, _, _ = reference_env(root, f.read())
            assert np.array_equal(bits(env), bits(g["env"])), name
        d = order - np.arange(n)
        assert np.abs(d).max() < 128
        out[name] = d.astype(np.int8)
    return out


def loader_records(reference):
    from tests import hdr_cases
    from tests.golden import make_texture_fixtures as mk
    from tests.golden.make_obj_fixtures import reference_env
    L = {}
    with tempfile.TemporaryDirectory() as tmp:
        for key, obj in H.loader_live_cases(tmp).items():
            L["obj/" + key] = H.scene_digests(refbind.RefRenderer().open_obj(reference, obj).scene())
        for i, (name, data) in enumerate(hdr_cases.cases(seed=31).items()):
            root = os.path.join(tmp, "env%d" % i); os.makedirs(root)
            L["env/" + name] = hdr_cases.digest(*reference_env(root, data))
    with tempfile.TemporaryDirectory() as tmp:
        names = H.loader_texture_images(tmp)
        L["textures/records"] = H.texture_record_digests(refbind.RefRenderer().open_obj(reference, H._textured_obj(pathlib.Path(tmp), names)).scene())
    with tempfile.TemporaryDirectory() as tmp:
        names = H.fresh_texture_files(tmp)
        for n, (w, h, texels) in mk.reference_texels(tmp, names).items():
            L["textures/fresh/" + n] = [int(w), int(h), digest(texels)]
    return L


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", default="/root/reference")
    a = ap.parse_args()
    if not refbind.available() or not refbind.available(libm=True):
        raise SystemExit("oracle/_ref/libref.so and libref_libm.so are needed: python oracle/build_ref.py --reference <tree>")
    out = os.path.join(HERE, "ref")
    os.makedirs(out, exist_ok=True)
    frames = oracle_vs_ref_frames()
    frames.update(generated_obj_frames(a.reference))
    for name, rec in (("frames.json.xz", frames), ("loader.json.xz", loader_records(a.reference))):
        with lzma.open(os.path.join(out, name), "wt", preset=9) as f:          # one case per line
            f.write("{\n" + ",\n".join(json.dumps(k) + ": " + json.dumps(rec[k], sort_keys=True, separators=(",", ":"))
                                        for k in sorted(rec)) + "\n}\n")
    np.savez_compressed(os.path.join(out, "libm_sample.npz"), **libm_samples())
    from raytracing_b200 import scene_io
    scene_io.save_npz_xz(os.path.join(REPO, "tests", "golden", "scenes", "input_order.npz.xz"), shipped_scene_orders(a.reference))
    print("wrote", os.path.relpath(out, REPO))
