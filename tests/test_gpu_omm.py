"""-m gpu parity with opacity micromaps (reference: src/gltf_scene_omm.cpp + docs/RENDERING_ARCHITECTURE.md:65-78): the traversal
kernels resolve OPAQUE / TRANSPARENT micro-triangles themselves (csrc/omm.cuh), only UNKNOWN ones reach the any-hit kernels.  The
checker is the oracle given the same micromap arrays."""
import numpy as np
import pytest

from conftest import rel_rmse
from gpu_util import trace_both
from test_gpu_scenes import _attach, _gpu_render, _oracle

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("level", [4, 3])
def test_trace_parity_with_baked_micromaps(std_env, oracle_mod, level):
    """Closest-hit and shadow rays through the production kernels on the foliage atrium with baked micromaps: committed hits,
    barycentrics and the per-ray seeds (one rand() per UNKNOWN candidate, none for resolved micro-triangles) bit-exact against the
    oracle holding the same micromaps -- and the hits equal the ones without micromaps while fewer seeds move."""
    from gpu_util import random_rays
    from vk_gltf_renderer_b200 import omm, synth
    scn = synth.synth_sponza(tex_size=256, detail=0.05)
    rays = random_rays(60000, [-15, 0, -6], [15, 12, 6])
    seeds = ((np.arange(len(rays), dtype=np.uint64) * 2654435761) % (2 ** 32)).astype(np.uint32)
    o0 = oracle_mod.Oracle()
    o0.set_scene(scn)
    s0 = seeds.copy()
    h0 = o0.trace_closest(rays, s0)
    st = omm.bake_opacity_micromaps(scn, level=level)
    assert st["triangles"] > 500 and st["opaque"] > 0 and st["transparent"] > 0
    pt, _ = _attach(scn, std_env, (16, 16))
    o = oracle_mod.Oracle()
    o.set_scene(scn)
    ref, s_ref, ref_t, _ = trace_both(pt, o, rays, seeds)
    assert np.array_equal(ref.view(np.uint32), h0.view(np.uint32))
    assert (s_ref != seeds).sum() < (s0 != seeds).sum()
    assert 0.02 < (ref_t[:, 0] > 0).mean() < 0.98


def deep_layers_with_micromaps():
    """14 MASK layers with level-3 micromaps, two of them mirrored, and 40 000 rays through them towards the back wall.
    Returns the scene, the bake statistics, the rays and their seeds."""
    from vk_gltf_renderer_b200 import omm, synth
    scn = synth.synth_layers(tex_size=256)
    # mirror two of the layers (negative determinant: the flattened record swaps its 2nd / 3rd vertex, TRI_FLIPPED)
    for rn in scn.render_nodes[2:4]:
        m = np.asarray(rn["objectToWorld"], np.float64).reshape(4, 4).T.copy()
        m = m @ np.diag([-1.0, 1.0, 1.0, 1.0])
        from vk_gltf_renderer_b200.scene import _glm
        rn["objectToWorld"], rn["worldToObject"] = _glm(m), _glm(np.linalg.inv(m))
    st = omm.bake_opacity_micromaps(scn, level=3)
    rng = np.random.default_rng(11)
    n = 40000
    rays = np.zeros((n, 8), np.float32)
    rays[:, 0:3] = np.stack([rng.uniform(-1.4, 1.4, n), rng.uniform(0.2, 2.0, n), rng.uniform(0.5, 3.0, n)], 1)
    tgt = np.stack([rng.uniform(-1.4, 1.4, n), rng.uniform(0.2, 2.0, n), np.full(n, -2.4)], 1)
    d = tgt - rays[:, 0:3]
    rays[:, 4:7] = d / np.linalg.norm(d, axis=1, keepdims=True)
    rays[:, 7] = 1e32
    seeds = ((np.arange(n, dtype=np.uint64) * 40503) % (2 ** 32)).astype(np.uint32)
    return scn, st, rays, seeds


def test_trace_parity_micromaps_on_deep_layers(std_env, oracle_mod):
    """14 MASK layers with micromaps: the few UNKNOWN candidates, OPAQUE micro-triangles committing in front of or behind them,
    continuation rounds behind a full candidate list -- closest and shadow, bit-exact, also on mirrored instances."""
    scn, st, rays, seeds = deep_layers_with_micromaps()
    assert st["unknown"] > 0.2 * st["micro"] and st["opaque"] > 0.03 * st["micro"] and st["transparent"] > 0.01 * st["micro"]
    pt, _ = _attach(scn, std_env, (16, 16))
    o = oracle_mod.Oracle()
    o.set_scene(scn)
    ref, s_ref, ref_t, ss_ref = trace_both(pt, o, rays, seeds, tmax=0.7)
    assert (s_ref != seeds).mean() > 0.1 and 0.01 < (ref_t[:, 0] > 0).mean() < 0.99 and (ss_ref != seeds).mean() > 0.01


def test_render_parity_with_baked_micromaps(std_env, oracle_mod):
    """The atrium rendered with micromaps: same tolerance as without (rel RMSE <= 1e-3 against the oracle with the same micromaps),
    the same pixels covered, and the any-hit kernels see fewer candidates."""
    from vk_gltf_renderer_b200 import omm, synth
    scn = synth.synth_sponza(tex_size=256, detail=0.05)
    pt0, img0 = _gpu_render(scn, std_env, 320, 180, 8, ptMaxDepth=6)
    omm.bake_opacity_micromaps(scn, level=4)
    o = _oracle(oracle_mod, scn, std_env)
    ref = oracle_mod.render(o, scn.camera, 320, 180, 8, max_depth=6)
    pt, img = _gpu_render(scn, std_env, 320, 180, 8, ptMaxDepth=6)
    assert np.isfinite(img).all()
    e = rel_rmse(img, ref)
    print("synth sponza + micromaps rel RMSE", e)
    assert e <= 1e-3
    assert np.array_equal(img[..., 3] > 0, img0[..., 3] > 0)
    assert abs(img[..., :3].mean() - img0[..., :3].mean()) / img0[..., :3].mean() < 0.02
    s0, s1 = pt0.stats(), pt.stats()
    assert s1["closestRays"] > 0.9 * s0["closestRays"]


def test_special_indices_and_two_state_format(std_env, oracle_mod):
    """hand-made micromaps: FULLY_OPAQUE / FULLY_TRANSPARENT special indices (no lookup, no any-hit work at all) and the 1-bit format
    at level 1 with only the centre micro-triangle opaque -- the same arrays tests/test_omm.py gives the oracle"""
    from vk_gltf_renderer_b200 import abi, synth
    scn = synth.synth_layers(layers=1, tex_size=32)
    pid = next(rn["renderPrimID"] for rn in scn.render_nodes if scn.materials[rn["materialID"]].alphaMode == 1)
    ntri = len(scn.render_prims[pid]["indices"])
    rng = np.random.default_rng(2)
    lo, hi = scn.bounds()
    rays = np.zeros((20000, 8), np.float32)
    rays[:, 0:3] = rng.uniform(lo - 0.5, hi + 0.5, (len(rays), 3))
    d = rng.normal(size=(len(rays), 3))
    rays[:, 4:7] = d / np.linalg.norm(d, axis=1, keepdims=True)
    rays[:, 7] = 1e30
    seeds = np.arange(len(rays), dtype=np.uint32)
    cases = [([dict(data=np.zeros(1, np.uint8), triangles=np.zeros(0, abi.MICROMAP_TRIANGLE_DTYPE))], np.full(ntri, sp, np.int32))
             for sp in (abi.OMM_INDEX_FULLY_OPAQUE, abi.OMM_INDEX_FULLY_TRANSPARENT, abi.OMM_INDEX_FULLY_UNKNOWN_OPAQUE)]
    cases.append(([dict(data=np.array([0b0010], np.uint8), triangles=np.array([(0, 1, abi.OMM_FORMAT_2_STATE)], abi.MICROMAP_TRIANGLE_DTYPE))], np.zeros(ntri, np.int32)))
    moved = []
    for mm, idx in cases:
        scn.micromaps, scn.prim_omms = mm, [dict(renderPrimID=pid, micromap=0, baseTriangle=0, indices=idx)]
        scn._keep = []
        pt, _ = _attach(scn, std_env, (16, 16))
        o = oracle_mod.Oracle()
        o.set_scene(scn)
        ref, s_ref, ref_t, ss_ref = trace_both(pt, o, rays, seeds, tmax=3.0)
        moved.append(int((s_ref != seeds).sum()))
        pt.onDetach()
    assert moved[0] == 0 and moved[1] == 0 and moved[2] > 100 and moved[3] == 0


def micromap_scene_and_bad_sets():
    """one foliage layer and micromap sets the library must refuse: a subdivision level above 12, data beyond dataSize, a linkage to
    a micromap, triangle or render primitive out of range, indices that do not cover the primitive"""
    from vk_gltf_renderer_b200 import abi, synth
    scn = synth.synth_layers(layers=1, tex_size=32)
    pid = next(rn["renderPrimID"] for rn in scn.render_nodes if scn.materials[rn["materialID"]].alphaMode == 1)
    ntri = len(scn.render_prims[pid]["indices"])
    return scn, [
        dict(mm=[dict(data=np.zeros(1, np.uint8), triangles=np.array([(0, 13, 2)], abi.MICROMAP_TRIANGLE_DTYPE))], po=[dict(renderPrimID=pid, micromap=0, indices=np.zeros(ntri, np.int32))]),
        dict(mm=[dict(data=np.zeros(1, np.uint8), triangles=np.array([(0, 3, 2)], abi.MICROMAP_TRIANGLE_DTYPE))], po=[dict(renderPrimID=pid, micromap=0, indices=np.zeros(ntri, np.int32))]),
        dict(mm=[dict(data=np.zeros(16, np.uint8), triangles=np.array([(0, 3, 2)], abi.MICROMAP_TRIANGLE_DTYPE))], po=[dict(renderPrimID=pid, micromap=1, indices=np.zeros(ntri, np.int32))]),
        dict(mm=[dict(data=np.zeros(16, np.uint8), triangles=np.array([(0, 3, 2)], abi.MICROMAP_TRIANGLE_DTYPE))], po=[dict(renderPrimID=pid, micromap=0, indices=np.full(ntri, 5, np.int32))]),
        dict(mm=[dict(data=np.zeros(16, np.uint8), triangles=np.array([(0, 3, 2)], abi.MICROMAP_TRIANGLE_DTYPE))], po=[dict(renderPrimID=pid, micromap=0, indices=np.zeros(1, np.int32))]),
        dict(mm=[dict(data=np.zeros(16, np.uint8), triangles=np.array([(0, 3, 2)], abi.MICROMAP_TRIANGLE_DTYPE))], po=[dict(renderPrimID=9999, micromap=0, indices=np.zeros(ntri, np.int32))]),
    ]


def test_micromap_arguments_are_validated(std_env):
    from vk_gltf_renderer_b200.renderer import B200PTError
    scn, bad = micromap_scene_and_bad_sets()
    for b in bad:
        scn.micromaps, scn.prim_omms = b["mm"], b["po"]
        with pytest.raises(B200PTError):
            _attach(scn, std_env, (16, 16))
    scn.micromaps, scn.prim_omms = [], []
    _attach(scn, std_env, (16, 16))


def test_cpp_host_hands_the_micromaps_over(std_env, tmp_path):
    """The scene blob carries the EXT_mesh_opacity_micromap arrays; the C++ host (SceneData + PathTracer::onSceneInvalidated) passes
    them to b200pt_set_opacity_micromaps unless --useOpacityMicromap 0 (src/main.cpp:114-115): the two headless images equal the
    Python host's renders with and without the arrays."""
    import os
    import subprocess
    from vk_gltf_renderer_b200 import _lib, omm, synth
    exe = os.path.join(os.path.dirname(_lib.LIB_PATH), "b200pt_headless")
    scn = synth.synth_sponza(tex_size=256, detail=0.05)
    _, ref_plain = _gpu_render(scn, std_env, 160, 96, 4, ptMaxDepth=5)
    omm.bake_opacity_micromaps(scn, level=4)
    _, ref_omm = _gpu_render(scn, std_env, 160, 96, 4, ptMaxDepth=5)
    assert not np.array_equal(ref_plain, ref_omm)
    blob = str(tmp_path / "atrium.b2sc")
    scn.save_blob(blob, std_env)
    for flag, ref in (("1", ref_omm), ("0", ref_plain)):
        raw = str(tmp_path / ("img%s.raw" % flag))
        out = subprocess.run([exe, "--scene", blob, "--size", "160", "96", "--frames", "4", "--ptMaxDepth", "5", "--useOpacityMicromap", flag, "--outRaw", raw],
                             capture_output=True, text=True, timeout=300)
        assert out.returncode == 0, out.stderr
        img = np.fromfile(raw, np.float32).reshape(96, 160, 4)
        # the two hosts compute the camera matrices independently (rounding of the frame constants flips a few silhouette paths on
        # this scene), so "equal" is relative to how far apart the two random streams are
        other = ref_plain if flag == "1" else ref_omm
        gap = rel_rmse(ref_omm, ref_plain)
        print("useOpacityMicromap", flag, "rel RMSE to its reference", rel_rmse(img, ref), "to the other", rel_rmse(img, other), "gap", gap)
        assert np.array_equal(img[..., 3] > 0, ref[..., 3] > 0)
        assert rel_rmse(img, ref) < 0.2 * gap and rel_rmse(img, other) > 0.6 * gap
