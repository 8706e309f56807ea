#!/usr/bin/env python3
"""
tests/golden/make_material_edge_records.py — what the REFERENCE's own kernels (oracle/_ref/libref.so, built by oracle/build_ref.py)
produce for the material-edge scenes of tests/material_cases.py, stored so that tests/test_material_edges_cpu.py pins the oracle to
them without the reference.

    python tests/golden/make_material_edge_records.py

Writes tests/golden/ref/material_edges.json.xz: per case and sample the per-bounce counters and the sha256 digests of the radiance
bits and primary hits (tests/helpers.frame_record), and per case the digest of the albedo AOV of its last sample.
"""
import json
import lzma
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, REPO)

from oracle import refbind  # noqa: E402
from tests import test_material_edges_cpu as T  # noqa: E402
from tests.golden.make_ref_records import ref_samples  # noqa: E402
from tests.helpers import bits, digest  # noqa: E402


def records():
    out = {}
    for key, (name, mb, n, wf, sampler) in T.REF_CASES.items():
        sc, cam, w, h = T.cached(name)
        tables = T.sampler_tables(sampler)
        out[key] = ref_samples(sc, cam, w, h, mb, n, wf, keys=T.REF_KEYS, tables=tables)
        r = refbind.RefRenderer().open_arrays(sc)
        r.begin(w, h); r.set_camera(cam); r.set_max_bounces(mb); r.enable_white_furnace(wf); r.enable_denoiser(True)
        if tables is not None:
            r.use_sampler_tables(tables); r.set_blue_noise(True)
        for _ in range(n):
            r.integrate()
        out[key + "/albedo"] = digest(bits(r.aov_albedo()[..., :3]))
        r.close()
    return out


if __name__ == "__main__":
    if not refbind.available():
        raise SystemExit("oracle/_ref/libref.so is needed: python oracle/build_ref.py --reference <tree>")
    rec = records()
    path = os.path.join(HERE, "ref", "material_edges.json.xz")
    with lzma.open(path, "wt", preset=9) as f:
        f.write("{\n" + ",\n".join(json.dumps(k) + ": " + json.dumps(rec[k], sort_keys=True, separators=(",", ":"))
                                    for k in sorted(rec)) + "\n}\n")
    print("wrote", os.path.relpath(path, REPO))
