"""The alpha-cap bake is conservative (-m "not gpu"): csrc/alpha_caps.cuh's capBakeCell -- the code k_cap_bake runs for every
micro-triangle -- is compiled for the host (tools/host_caps_check.cpp) and run on the alpha records of real scenes.  For every
micro-triangle it marks as a cap, the oracle's level-0 sampler (sampleLevel0, what getOpacity reads) must give opacity exactly 1 at
dense points inside it, on its edges and at its corners, with the hit-side fp32 arithmetic of opacityFromRecord: uv interpolated from
w = 1 - u - v, texel alpha x factor x interpolated vertex-colour alpha, then the MASK cutoff (or exactly 1 for BLEND).  The records
cover every sampler state of synth.sampler_layers (REPEAT / CLAMP_TO_EDGE / MIRRORED_REPEAT per axis, NEAREST and LINEAR,
non-power-of-two, N x 1 and 1 x N images, uv far outside [0, 1], TEXCOORD_1, specular-glossiness, vertex-colour alpha, BLEND) with
their own and with moved factors and cutoffs, and the foliage atlas of SynthSponza as MASK and as nearest-filtered BLEND."""
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "vk_gltf_renderer_b200", "csrc")
CUDA_INC = os.environ.get("CUDA_HOME", "/usr/local/cuda") + "/include"
LEVEL = 5
NEAREST = (9728, 9984, 9986)


@pytest.fixture(scope="module")
def checker(tmp_path_factory):
    if not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")):
        pytest.skip("CUDA headers not found")
    exe = str(tmp_path_factory.mktemp("capcheck") / "host_caps_check")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I" + CUDA_INC, "-o", exe, os.path.join(CSRC, "tools", "host_caps_check.cpp")])
    return exe


def _records(scn):
    """(record fields, texture-info slot, vertex uv of the sampled set, vertex-colour alphas) of every alpha-tested triangle"""
    out = []
    for rn in scn.render_nodes:
        m = scn.materials[max(rn["materialID"], 0)]
        if m.alphaMode == 0:
            continue
        p = scn.render_prims[rn["renderPrimID"]]
        spec = m.pbrModel == 1
        slot = m.pbrDiffuseTexture if spec else m.pbrBaseColorTexture
        factor = m.pbrDiffuseFactor[3] if spec else m.pbrBaseColorFactor[3]
        ti = scn.texture_infos[slot] if slot > 0 else None
        tex = scn.textures[ti.index] if ti is not None else None
        uvs = (p["uv1"] if ti.texCoord else p["uv0"]) if ti is not None else None
        for tri in p["indices"]:
            uv = uvs[tri].astype(np.float32) if uvs is not None else np.zeros((3, 2), np.float32)
            col = None if p["colors"] is None else (p["colors"][tri] >> 24).astype(np.uint32)
            mode = m.alphaMode | (4 if tex is not None and tex["magFilter"] not in NEAREST else 0) | (8 if col is not None else 0)
            out.append(dict(uv=uv, tex=tex, slot=slot, factor=np.float32(factor), cutoff=np.float32(m.alphaCutoff), mode=mode, col=col))
    return out


def _bake(exe, recs, path):
    with open(path + ".in", "wb") as f:
        f.write(np.uint32(len(recs)).tobytes())
        for r in recs:
            t = r["tex"]
            h, w = (t["rgba8"].shape[:2]) if t is not None else (0, 0)
            colA = 0 if r["col"] is None else int(r["col"][0] | (r["col"][1] << 8) | (r["col"][2] << 16))
            f.write(r["uv"].reshape(-1).tobytes())
            f.write(np.array([w, h, t["wrapS"] if t else 0, t["wrapT"] if t else 0], np.int32).tobytes())
            f.write(np.array([r["factor"], r["cutoff"]], np.float32).tobytes())
            f.write(np.array([r["mode"], colA, 1 if t is not None else 0], np.uint32).tobytes())
            if t is not None:
                f.write(np.ascontiguousarray(t["rgba8"][..., 3]).tobytes())
    subprocess.check_call([exe, path + ".in", path + ".out"])
    words = np.fromfile(path + ".out", np.uint32).reshape(len(recs), -1)
    return np.unpackbits(words.view(np.uint8), bitorder="little").reshape(len(recs), -1).astype(bool)


def _dense_points(corners, steps=6):
    """barycentric (u, v) float32 of a lattice over each micro-triangle, corners and edges included: [cells, points, 2]"""
    ab = np.array([(a, b) for a in range(steps + 1) for b in range(steps + 1 - a)], np.float64) / steps
    c = corners[:, None]
    return (c[..., 0, :] + ab[None, :, 0:1] * (c[..., 1, :] - c[..., 0, :]) + ab[None, :, 1:2] * (c[..., 2, :] - c[..., 0, :])).astype(np.float32)


def _check(exe, o, scn, recs, tmp_path, tag):
    from vk_gltf_renderer_b200 import omm
    caps = _bake(exe, recs, str(tmp_path / tag))
    corners = omm.micro_triangle_corners(LEVEL)
    total = 0
    for r, cap in zip(recs, caps):
        if not cap.any():
            continue
        pts = _dense_points(corners[cap]).reshape(-1, 2)
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
        ok = a >= r["cutoff"] if (r["mode"] & 3) == 1 else a == np.float32(1)
        assert ok.all(), (tag, r["mode"], r["factor"], r["cutoff"], pts[~ok][:4], a[~ok][:4])
        total += int(cap.sum())
    return total, caps.size


def test_bake_is_conservative_on_sampler_layers(checker, oracle_mod, tmp_path):
    from vk_gltf_renderer_b200 import synth
    scn = synth.sampler_layers()
    o = oracle_mod.Oracle()
    o.set_scene(scn)
    recs = _records(scn)
    assert len({r["mode"] for r in recs}) >= 4
    found = 0
    for factor_scale, cutoff in ((1.0, None), (0.8, None), (1.0, 0.2), (1.25, 0.9), (0.5, 0.0)):
        rs = [dict(r, factor=np.float32(r["factor"] * factor_scale), cutoff=r["cutoff"] if cutoff is None else np.float32(cutoff)) for r in recs]
        n, _ = _check(checker, o, scn, rs, tmp_path, f"layers_{factor_scale}_{cutoff}")
        found += n
    assert found > 1000, found


def test_bake_is_conservative_on_the_foliage_atlas(checker, oracle_mod, tmp_path):
    """the leaf atlas (binary ellipse mask, 4 x 4 cells) on quads over every cell, under REPEAT, CLAMP_TO_EDGE and MIRRORED_REPEAT, also
    shifted by whole texture periods far outside [0, 1]; MASK with linear filtering and BLEND with nearest filtering"""
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
    n, cells = _check(checker, o, scn, recs, tmp_path, "leaves")
    # the ellipse covers ~37 % of a cell; the bake must find most of its interior
    assert n > 0.2 * cells, (n, cells)
