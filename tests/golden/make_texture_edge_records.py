#!/usr/bin/env python3
"""
tests/golden/make_texture_edge_records.py — what the REFERENCE's own kernels (oracle/_ref/libref.so, built by oracle/build_ref.py)
produce for the texture-chart and emission-ladder scenes of tests/texture_cases.py, stored so that
tests/test_texture_edges_cpu.py pins the oracle to them without the reference.

    python tests/golden/make_texture_edge_records.py

Writes tests/golden/ref/texture_edges.json.xz: per case and sample the per-bounce counters and the sha256 digests of the
radiance bits and primary hits (tests/helpers.frame_record), and per chart the digest of the bounce-0 albedo AOV.
"""
import json
import lzma
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, REPO)

from oracle import refbind  # noqa: E402
from tests import test_texture_edges_cpu as T  # noqa: E402
from tests.golden.make_ref_records import ref_samples  # noqa: E402
from tests.helpers import bits, digest  # noqa: E402


def records():
    out = {}
    for key, (build, cam, w, h, mb, n) in T.REF_CASES.items():
        sc = build()
        out[key] = ref_samples(sc, cam(w, h), w, h, mb, n, keys=T.REF_KEYS)
        if key.startswith("chart"):
            r = refbind.RefRenderer().open_arrays(sc)
            r.begin(w, h); r.set_camera(cam(w, h)); r.set_max_bounces(mb); r.enable_denoiser(True); r.integrate()
            out[key + "/albedo"] = digest(bits(r.aov_albedo()[..., :3]))
            r.close()
    return out


if __name__ == "__main__":
    if not refbind.available():
        raise SystemExit("oracle/_ref/libref.so is needed: python oracle/build_ref.py --reference <tree>")
    rec = records()
    path = os.path.join(HERE, "ref", "texture_edges.json.xz")
    with lzma.open(path, "wt", preset=9) as f:
        f.write("{\n" + ",\n".join(json.dumps(k) + ": " + json.dumps(rec[k], sort_keys=True, separators=(",", ":"))
                                    for k in sorted(rec)) + "\n}\n")
    print("wrote", os.path.relpath(path, REPO))
