"""-m gpu parity of the animation feed (b200pt_set_animation / b200pt_animate): the morph and skinning kernels
(shaders/morph.comp.slang, shaders/skinning.comp.slang as SceneAnimationVk::cmdUpdateAnimation dispatches them,
src/gltf_scene_animation_vk.cpp:396-592) write the primitives' vertex arrays on the device, the shade records are re-gathered
and the trees refitted; the oracle (oracle/animation.py + the path-tracer oracle on the deformed scene, built from scratch)
must see the same geometry: ray-level hits bit for bit, images to 1e-3."""
import copy

import numpy as np
import pytest

from conftest import rel_rmse

pytestmark = pytest.mark.gpu


def _check_pose(pt, res, scn_ref, std_env, oracle_mod, tag, frames=4):
    import torch
    from gpu_util import random_rays, to_dev
    o = oracle_mod.Oracle()
    o.set_scene(scn_ref)
    o.set_environment(std_env)
    rays = random_rays(40000, [-3.5, 0, -2.5], [3.5, 3.2, 2.5], seed=21)
    ref = o.trace_closest(rays)
    d_rays = to_dev(rays)
    d_hits = torch.empty((len(rays), 6), dtype=torch.float32, device="cuda")
    pt.trace_closest(d_rays.data_ptr(), len(rays), d_hits.data_ptr())
    pt.synchronize()
    got = d_hits.cpu().numpy()
    assert (ref.view(np.uint32)[:, 1] != 0xFFFFFFFF).mean() > 0.3
    assert np.array_equal(got.view(np.uint32)[:, 1:4], ref.view(np.uint32)[:, 1:4]), tag   # node, primitive, triangle ids
    assert np.array_equal(got[:, [0, 4, 5]], ref[:, [0, 4, 5]]), tag                        # t, u, v: the positions are bit-identical
    rays[:, 7] = 2.5
    ref_t = o.trace_shadow(rays)
    d_rays = to_dev(rays)
    d_t = torch.empty((len(rays), 3), dtype=torch.float32, device="cuda")
    pt.trace_shadow(d_rays.data_ptr(), len(rays), d_t.data_ptr())
    pt.synchronize()
    assert np.array_equal(d_t.cpu().numpy(), ref_t), tag
    img_ref = oracle_mod.render(o, scn_ref.camera, 160, 112, frames, max_depth=5)
    for f in range(frames):
        res.frameCount = f
        pt.onRender(None, res)
    img = pt.read_accum()
    e = rel_rmse(img, img_ref)
    print(tag, "rel RMSE", e)
    assert np.isfinite(img).all() and e <= 1e-3, (tag, e)   # shading reads the skinned / morphed normals and tangents (normal maps)
    return img


@pytest.mark.parametrize("builder", [0, 1])
def test_morph_and_skin_on_the_device_match_the_oracle(std_env, oracle_mod, builder):
    """Three poses in sequence on one handle (rest, bent + bulged, bent the other way): every b200pt_animate starts from the
    static base arrays (or, for the banner, from its freshly morphed arrays), so the result never depends on the previous pose.
    builder 1: the trees being refitted were built on the device (LBVH)."""
    from oracle import animation as A
    from vk_gltf_renderer_b200 import synth
    from vk_gltf_renderer_b200.renderer import PathTracer, Resources
    scn, morphs, skins, pose = synth.synth_animated()
    rest = synth.scene_from_state(copy.deepcopy(synth.scene_state(scn)))
    res = Resources(scene=scn, hdr_rgb=std_env, camera=scn.camera, size=(160, 112))
    pt = PathTracer(0)
    pt.ptMaxDepth = 5
    pt.onAttach(res)
    if builder:
        pt.set_bvh_builder(builder)
        pt.onSceneInvalidated(res)
    pt.set_animation(morphs, skins)
    imgs = []
    for k in (1, 2, 0):
        mw, jm, nm = pose(k)
        pt.animate(mw, jm, nm)
        ref_scn = synth.scene_from_state(copy.deepcopy(synth.scene_state(rest)))
        A.apply(ref_scn, morphs, skins, mw, jm, nm)
        imgs.append(_check_pose(pt, res, ref_scn, std_env, oracle_mod, "builder %d pose %d" % (builder, k)))
    # the poses differ visibly (the feed does something), and pose 0 is the rest pose up to normalisation
    assert rel_rmse(imgs[0], imgs[1]) > 0.02 and rel_rmse(imgs[0], imgs[2]) > 0.02
    pt.onDetach(res)


def test_animation_argument_checks(std_env):
    """b200pt_set_animation before a scene, a vertex count that is not the primitive's, a primitive out of range, b200pt_animate
    without tasks: B200PT_E_INVALID, never an out-of-bounds access."""
    from vk_gltf_renderer_b200 import synth
    from vk_gltf_renderer_b200.animation import MorphTask
    from vk_gltf_renderer_b200.renderer import B200PTError, PathTracer, Resources
    scn, morphs, skins, pose = synth.synth_animated()
    res = Resources(scene=scn, hdr_rgb=std_env, camera=scn.camera, size=(64, 48))
    pt = PathTracer(0)
    pt.onAttach(res)
    with pytest.raises(B200PTError):
        pt.animate(*pose(1))                       # no tasks yet
    bad = copy.deepcopy(morphs[0])
    bad.base_positions = bad.base_positions[:-3]
    bad.position_deltas = bad.position_deltas[:, :-3]
    with pytest.raises(B200PTError):
        pt.set_animation([bad], [])
    far = copy.deepcopy(skins[0])
    far.render_prim = 99
    with pytest.raises(B200PTError):
        pt.set_animation([], [far])
    pt.set_animation(morphs, skins)
    pt.animate(*pose(2))
    with pytest.raises(B200PTError):
        pt.set_animation(morphs, [far])            # a refused set_animation leaves no tasks, not the previous ones
    with pytest.raises(B200PTError):
        pt.animate(*pose(1))
    pt.set_animation(morphs, skins)
    pt.onSceneInvalidated(res)                     # a new scene drops the tasks
    with pytest.raises(B200PTError):
        pt.animate(*pose(1))
    pt.onDetach(res)


def test_node_hierarchy_on_the_device_matches_the_oracle(std_env, oracle_mod):
    """b200pt_set_node_hierarchy / b200pt_update_node_matrices: local matrices go up, world matrices are propagated level by level
    on the device, the render nodes (objectToWorld, inverse, ids) rewritten and the trees refitted.  The oracle builds the scene
    from scratch with the render nodes oracle/animation.py computes: hits bit for bit, image to 1e-3 (the inverse feeds the
    normals).  One node chain mirrors its instance (negative determinant: the refit flips the winding)."""
    from oracle import animation as A
    from vk_gltf_renderer_b200 import synth
    from vk_gltf_renderer_b200.animation import topo_levels
    from vk_gltf_renderer_b200.renderer import B200PTError, PathTracer, Resources
    scn, parents, mappings, inst, pose = synth.synth_hierarchy()
    glm = lambda ms: np.ascontiguousarray(np.asarray(ms, np.float64).transpose(0, 2, 1).astype(np.float32))
    res = Resources(scene=scn, hdr_rgb=std_env, camera=scn.camera, size=(160, 112))
    pt = PathTracer(0)
    pt.ptMaxDepth = 5
    pt.onAttach(res)
    with pytest.raises(B200PTError):
        pt.update_node_matrices(glm(pose(0)))          # no hierarchy yet
    pt.set_node_hierarchy(parents, mappings, glm(inst))
    order, offsets = topo_levels(parents)
    for k in (1, 2, 0):
        loc = glm(pose(k))
        pt.update_node_matrices(loc)
        o2w, w2o = A.render_nodes(A.propagate(loc, parents, order, offsets), mappings, glm(inst))
        ref_scn = synth.scene_from_state(copy.deepcopy(synth.scene_state(scn)))
        for i, rn in enumerate(ref_scn.render_nodes):
            rn["objectToWorld"], rn["worldToObject"] = o2w[i].reshape(-1).copy(), w2o[i].reshape(-1).copy()
        _check_pose(pt, res, ref_scn, std_env, oracle_mod, "hierarchy pose %d" % k)
    bad = parents.copy()
    bad[1], bad[2] = 2, 1                               # a cycle: no valid level order
    with pytest.raises(ValueError):
        pt.set_node_hierarchy(bad, mappings)
    far = [(len(parents), mat, prim) for _, mat, prim in mappings]   # every render node mapped to a node out of range
    with pytest.raises(B200PTError):
        pt.set_node_hierarchy(parents, far)
    with pytest.raises(B200PTError):
        pt.update_node_matrices(glm(pose(1)))          # the refused hierarchy left none
    pt.onDetach(res)
