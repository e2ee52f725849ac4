"""The alpha-hole bake is conservative (-m "not gpu"): csrc/alpha_caps.cuh's capBakeCell, compiled for the host
(tools/host_caps_check.cpp ... holes), marks micro-triangles whose opacity is exactly 0 everywhere.  For every one of them the oracle's
level-0 sampler must give opacity exactly 0 at dense points inside it, on its edges and at its corners, with the hit-side fp32 arithmetic
of opacityFromRecord (as tests/test_alpha_caps.py checks the caps), on every sampler state of synth.sampler_layers with moved factors and
cutoffs and on the foliage atlas of SynthSponza; and no micro-triangle is both a cap and a hole."""
import subprocess

import numpy as np

from test_alpha_caps import LEVEL, NEAREST, _bake, _dense_points, _records, checker  # noqa: F401 (checker: the fixture)


def _bake_both(exe, recs, path):
    caps = _bake(exe, recs, path)
    subprocess.check_call([exe, path + ".in", path + ".holes", "holes"])
    words = np.fromfile(path + ".holes", np.uint32).reshape(len(recs), -1)
    return caps, np.unpackbits(words.view(np.uint8), bitorder="little").reshape(len(recs), -1).astype(bool)


def _check(exe, o, recs, tmp_path, tag):
    from vk_gltf_renderer_b200 import omm
    caps, holes = _bake_both(exe, recs, str(tmp_path / tag))
    assert not (caps & holes).any()
    corners = omm.micro_triangle_corners(LEVEL)
    total = 0
    for r, hole in zip(recs, holes):
        if not hole.any():
            continue
        pts = _dense_points(corners[hole]).reshape(-1, 2)
        u, v = pts[:, 0], pts[:, 1]
        w = np.float32(1) - u - v
        uv = r["uv"]
        a = np.full(len(pts), r["factor"], np.float32)
        if r["tex"] is not None:
            tc = (uv[0] * w[:, None] + uv[1] * u[:, None]) + uv[2] * v[:, None]
            rec = np.zeros((len(pts), 8), np.float32)
            rec[:, 0], rec[:, 1], rec[:, 2:4], rec[:, 4:6] = r["slot"], 1, tc, tc
            a = a * o.texture_lookup(rec)[:, 3]
        if r["col"] is not None:
            ca = r["col"].astype(np.float32) / np.float32(255)
            a = a * ((ca[0] * w + ca[1] * u) + ca[2] * v)
        ok = a < r["cutoff"] if (r["mode"] & 3) == 1 else a == np.float32(0)
        assert ok.all(), (tag, r["mode"], r["factor"], r["cutoff"], pts[~ok][:4], a[~ok][:4])
        total += int(hole.sum())
    return total, holes.size


def test_hole_bake_is_conservative_on_sampler_layers(checker, oracle_mod, tmp_path):  # noqa: F811
    from vk_gltf_renderer_b200 import synth
    scn = synth.sampler_layers()
    o = oracle_mod.Oracle()
    o.set_scene(scn)
    recs = _records(scn)
    found = 0
    for factor_scale, cutoff in ((1.0, None), (0.8, None), (1.0, 0.2), (1.25, 0.9), (0.5, 0.0), (0.0, None)):
        rs = [dict(r, factor=np.float32(r["factor"] * factor_scale), cutoff=r["cutoff"] if cutoff is None else np.float32(cutoff)) for r in recs]
        n, _ = _check(checker, o, rs, tmp_path, f"layers_{factor_scale}_{cutoff}")
        found += n
    assert found > 1000, found


def test_hole_bake_is_conservative_on_the_foliage_atlas(checker, oracle_mod, tmp_path):  # noqa: F811
    """the leaf atlas on quads over every cell, REPEAT / CLAMP_TO_EDGE / MIRRORED_REPEAT, MASK linear and BLEND nearest"""
    from vk_gltf_renderer_b200 import synth
    from vk_gltf_renderer_b200.scene import Scene
    rng = np.random.default_rng(5)
    img = synth.make_leaf_texture(128, rng)
    scn = Scene()
    recs = []
    for ws, wt, mag, mode in ((10497, 10497, 9729, 1), (33071, 33648, 9729, 1), (33648, 10497, 9728, 2)):
        tex = scn.add_texture(img, srgb=True, wrapS=ws, wrapT=wt, magFilter=mag)
        slot = scn.add_texture_info(tex, 0)
        for cx in range(4):
            for cy in range(4):
                shift = np.float32(rng.integers(-6, 7)) if ws == 10497 else np.float32(0)
                c = np.array([cx, cy], np.float32) * np.float32(0.25) + shift
                quad = np.array([c, c + [0.25, 0], c + [0.25, 0.25], c + [0, 0.25]], np.float32)
                for tri in ((0, 1, 2), (0, 2, 3)):
                    recs.append(dict(uv=quad[list(tri)], tex=scn.textures[tex], slot=slot, factor=np.float32(1), cutoff=np.float32(0.5),
                                     mode=mode | (4 if mag not in NEAREST else 0), col=None))
    scn.add_material()
    o = oracle_mod.Oracle()
    o.set_scene(scn)
    n, cells = _check(checker, o, recs, tmp_path, "leaves")
    # outside the ellipse (~63 % of a cell) the atlas is transparent; the bake must find most of it
    assert n > 0.3 * cells, (n, cells)
