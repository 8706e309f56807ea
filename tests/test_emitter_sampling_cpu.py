"""
Emitter sampling (RT_OPT_EMITTER_SAMPLING) on the CPU: the emitter table every upload builds (raytracing_b200/csrc/rt_emitters.h)
against a numpy restatement, the inactive cases against the oracle, and the estimator's expectation against the oracle's.
"""
import os

import numpy as np
import pytest

from raytracing_b200 import hostapi
from raytracing_b200.camera import default_camera
from tests.emitter_model import EmitterModel
from tests.helpers import bits, scene

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PROC_OBJ = os.path.join(REPO, "tests", "golden", "scenes", "procedural.obj")


def procedural_scene():
    """The generated scene: a rough dielectric floor, a pass-through sheet, rough metal, a mirror and the emissive lamp."""
    s = hostapi.HostScene(PROC_OBJ)
    s.add_directional_light((-0.6, -1.5, 3.5), (15, 10, 5))
    s.build_bvh()
    s.finalize(env=np.full(4, 0.2, dtype=np.float32), env_width=1, env_height=1)
    a = s.arrays()
    s.close()
    return a


def get_scene(name):
    return procedural_scene() if name == "procedural" else scene(name)


def numpy_table(sc):
    """The rule of rt_emitters.h restated in numpy float32."""
    f = np.float32
    idx = np.asarray(sc["emissive"], dtype=np.int64)
    tris = sc["triangles"]
    mats = sc["materials"]
    p = [np.stack([tris[v]["position"][:, k] for k in range(3)], 1).astype(f) for v in ("v1", "v2", "v3")]
    e1, e2 = p[1] - p[0], p[2] - p[0]
    c = np.stack([e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1], e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2], e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]], 1)
    area = f(0.5) * np.sqrt((c[:, 0] * c[:, 0] + c[:, 1] * c[:, 1]) + c[:, 2] * c[:, 2])
    em = mats["emission"].astype(np.uint32)
    scale = np.ldexp(np.ones(len(em), f), (em >> 24).astype(np.int32) - 136).astype(f)
    rgb = [((em >> s) & 0xFF).astype(f) * scale for s in (0, 8, 16)]
    luma = (rgb[0] * f(0.299) + rgb[1] * f(0.587)) + rgb[2] * f(0.114)
    w = (area[idx] * luma[tris["mtlIndex"][idx]]).astype(f)
    w = np.where(np.isfinite(w) & (w > 0), w, f(0))
    s = f(0)
    run = []
    for x in w:
        s = f(s + x)
        run.append(s)
    cdf = (np.array(run, f) / s).astype(f)
    cdf[-1] = 1
    pmf = (cdf - np.concatenate([[f(0)], cdf[:-1]])).astype(f)
    pe = f(1.0) if not np.any(sc["lights"]["radiance"][:, :3] != 0) else f(0.5)
    pdfa = np.zeros(len(tris), f)
    pdfa[idx] = np.where(pmf > 0, (pe * pmf) / area[idx], f(0))
    return idx.astype(np.uint32), cdf, pdfa, pe


@pytest.mark.parametrize("name", ["CornellBox", "ShaderBalls", "procedural"])
def test_table_matches_numpy_restatement(name):
    sc = get_scene(name)
    m = EmitterModel(sc)
    lst, cdf, pdfa, pe = m.table()
    e_lst, e_cdf, e_pdfa, e_pe = numpy_table(sc)
    assert len(sc["emissive"]) > 0
    assert np.array_equal(lst, np.asarray(sc["emissive"], "<u4"))
    assert np.all(np.diff(cdf) >= 0) and cdf[-1] == 1.0
    assert pe == e_pe == 0.5
    assert np.array_equal(bits(cdf), bits(e_cdf))
    assert np.array_equal(bits(pdfa), bits(e_pdfa))
    off = np.ones(len(pdfa), bool); off[lst] = False
    assert np.all(pdfa[off] == 0) and np.all(pdfa[lst] > 0)
    assert m.table(white_furnace=True)[3] == 0.0


def test_table_rejects_bad_lists_and_handles_dark_lights():
    sc = dict(scene("CornellBox"))
    n = len(sc["triangles"])
    assert EmitterModel(sc, emissive=[0, 1, 0]).table() is None
    assert EmitterModel(sc, emissive=[n]).table() is None
    dark = dict(sc); dark["lights"] = sc["lights"].copy(); dark["lights"]["radiance"] = 0
    assert EmitterModel(dark).table()[3] == 1.0
    t = EmitterModel(sc, emissive=[]).table()
    assert t[3] == 0.0 and len(t[0]) == 0


@pytest.mark.parametrize("case", ["no_emitters", "white_furnace"])
def test_inactive_is_byte_identical_to_off(case):
    sc = scene("CornellBox")
    m = EmitterModel(sc, emissive=[] if case == "no_emitters" else None)
    wf = case == "white_furnace"
    w, h = 24, 16
    cam = default_camera(w, h)
    for s in range(2):
        a, _, sa = m.render(cam, w, h, 3, s, white_furnace=wf)
        b, _, sb = m.render(cam, w, h, 3, s, white_furnace=wf, emitters=True)
        assert np.array_equal(bits(a), bits(b))
        assert sa.tobytes() == sb.tobytes()


def batch_means(m, cam, w, h, mb, n, batches, emitters, first=0):
    """Per-batch mean images of samples first .. first + n - 1, and the per-pixel variance of one sample."""
    out = np.zeros((batches, h, w, 3), np.float64)
    per = n // batches
    sq = np.zeros((h, w, 3), np.float64)
    for b in range(batches):
        acc = np.zeros((h, w, 3), np.float64)
        for s in range(first + b * per, first + (b + 1) * per):
            r = m.render(cam, w, h, mb, s, emitters=emitters)[0][..., :3].astype(np.float64)
            acc += r
            sq += r * r
        out[b] = acc / per
    mean = out.mean(0)
    return out, sq / n - mean * mean


@pytest.mark.parametrize("name", ["procedural", "CornellBox"])
def test_same_expectation_as_the_oracle(name):
    """Per 8x8 tile and channel, z = (m_on - m_off) / sqrt(se_on^2 + se_off^2) with batch-mean standard errors."""
    sc = get_scene(name)
    m = EmitterModel(sc)
    w = h = 32
    cam = default_camera(w, h)
    n, batches = 2000, 20
    # the arms use disjoint sample indices, so that they are independent estimates
    on, var_on = batch_means(m, cam, w, h, 3, n, batches, True)
    off, var_off = batch_means(m, cam, w, h, 3, n, batches, False, first=n)
    tile = lambda x: x.reshape(x.shape[0], h // 8, 8, w // 8, 8, 3).mean((2, 4))
    ton, toff = tile(on), tile(off)
    se = lambda t: t.std(0, ddof=1) / np.sqrt(batches)
    # tiles without noise (the sky seen directly) differ only by the rounding of the float accumulations, which is about 2e-4 of
    # their value after 16 K samples: tiles whose standard error is below 3e-4 of their value are left out
    var = se(ton) ** 2 + se(toff) ** 2
    z = (ton.mean(0) - toff.mean(0)) / np.sqrt(var)
    z = z[np.isfinite(z) & (np.sqrt(var) > 3e-4 * np.abs(toff.mean(0)))]
    assert z.size > 0
    print("%s: %d tiles x channels, max |z| %.2f, mean z^2 %.2f; mean per-pixel variance on %.4g, off %.4g"
          % (name, z.size, np.abs(z).max(), np.mean(z * z), var_on.mean(), var_off.mean()))
    assert np.all(np.abs(z) < 5)
    assert 0.5 <= np.mean(z * z) <= 2.0
    if name == "CornellBox":
        # lit mainly by its ceiling emitter: the noise falls.  The procedural scene is lit mainly by its directional light, which
        # P_e = 1/2 samples half as often (at twice the weight), and its per-pixel variance rises; the print above records it.
        assert var_on.mean() < var_off.mean()
