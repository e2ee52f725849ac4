"""-m gpu KHR_animation_pointer playback: the clip of tests/test_animation_pointer.py played on one handle through
animation.sample_pointers / apply_pointers and PathTracer.update_scene_changes, next to the TRS / weights feed
(update_node_matrices, animate).  At every time the handle renders what a fresh handle renders when b200pt_set_scene gets the
sampled description and the same animation calls: image, selection ids and depth, and ray counters bit for bit, with either
BVH builder.  The device matches the oracle's image of the posed, sampled scene to 1e-3."""
import copy

import numpy as np
import pytest

from conftest import rel_rmse

pytestmark = pytest.mark.gpu

SIZE = (96, 72)
FRAMES = 3
STATS = ("closestRays", "shadowRays", "shadedHits", "pathsStarted")
# 0.37 -> 1.0: the transmission step (the trees are rebuilt) and the alpha-cutoff step (the alpha caps are re-baked); 1.0 again:
# nothing is sent; 1.6: the parent is shown (rebuilt); 2.5: past every key, the loaded description again
TIMES = (0.0, 0.37, 1.0, 1.0, 1.6, 2.0, 2.5)
ORACLE_TIMES = (0.37, 1.6)


def _glm(locals_):
    return np.ascontiguousarray(np.asarray(locals_, np.float64).transpose(0, 2, 1).astype(np.float32))


def _clone(scn):
    from vk_gltf_renderer_b200 import synth
    c = synth.scene_from_state(copy.deepcopy(synth.scene_state(scn)))
    c.graph = scn.graph
    return c


def _attach(scn, env, builder):
    from vk_gltf_renderer_b200.renderer import PathTracer, Resources
    res = Resources(scene=scn, hdr_rgb=env, camera=scn.camera, size=SIZE)
    pt = PathTracer(0)
    pt.ptMaxDepth = 5
    pt.onAttach(res)
    if builder:
        pt.set_bvh_builder(builder)
        pt.onSceneInvalidated(res)
    return pt, res


def _feed(pt, scn, tasks, time, first=False):
    """the TRS / weights half of the clip at `time`: node matrices and morph weights"""
    from vk_gltf_renderer_b200 import animation as anim
    morphs, skins = tasks
    if first:
        parents, mappings, inst = anim.node_hierarchy(scn)
        pt.set_node_hierarchy(parents, mappings, inst)
        pt.set_animation(morphs, skins)
    locals_, mesh_weights = anim.sample_animation(scn, 0, time)
    weights, jm, nm = anim.frame_inputs(scn, morphs, skins, locals_, mesh_weights)
    pt.update_node_matrices(_glm(locals_))
    pt.animate(weights, jm, nm)
    return locals_, weights


def _snapshot(pt, res):
    pt.reset_stats()
    for f in range(FRAMES):
        res.frameCount = f
        pt.onRender(None, res)
    pt.flush()
    pt.synchronize()
    out = dict(img=pt.read_accum())
    out["ids"], out["depth"] = pt.read_selection()
    st = pt.stats()
    out["stats"] = [st[k] for k in STATS]
    return out


def _oracle_image(oracle_mod, scn, tasks, locals_, weights, env):
    from oracle import animation as A
    from vk_gltf_renderer_b200 import animation as anim
    ref = _clone(scn)
    A.apply(ref, tasks[0], tasks[1], weights, [], [])
    parents, mappings, inst = anim.node_hierarchy(scn)
    order, offsets = anim.topo_levels(parents)
    o2w, w2o = A.render_nodes(A.propagate(_glm(locals_), parents, order, offsets), mappings, inst)
    for i, rn in enumerate(ref.render_nodes):
        rn["objectToWorld"], rn["worldToObject"] = o2w[i].reshape(-1).copy(), w2o[i].reshape(-1).copy()
    o = oracle_mod.Oracle()
    o.set_scene(ref)
    o.set_environment(env)
    img = oracle_mod.render(o, scn.camera, SIZE[0], SIZE[1], FRAMES, max_depth=5)
    o.close()
    return img


@pytest.mark.parametrize("builder", [0, 1])
def test_pointer_clip_on_one_handle_matches_fresh_handles(tmp_path, std_env, oracle_mod, builder):
    from test_animation_pointer import write_asset
    from vk_gltf_renderer_b200 import animation as anim, scene
    scn = scene.load_gltf(write_asset(tmp_path / "pointer.gltf"))
    tasks = anim.tasks_from_scene(scn)
    assert len(tasks[0]) == 1
    pt, res = _attach(scn, std_env, builder)
    sent = []
    for name in ("update_materials", "update_lights", "set_node_visibility"):
        def counted(r, f=getattr(pt, name), name=name):
            sent.append(name)
            f(r)
        setattr(pt, name, counted)
    prev = None
    for k, time in enumerate(TIMES):
        anim.apply_pointers(scn, *anim.sample_pointers(scn, 0, time))
        before, ms = len(sent), pt.bvh_build_ms()
        pt.update_scene_changes(res)
        edits = sent[before:]
        if time == prev:
            assert edits == [], (time, edits)                      # a repeated time sends nothing
        if (prev, time) == (0.0, 0.37):
            assert edits == ["update_materials", "update_lights"] and pt.bvh_build_ms() == ms     # values only: in place
        if (prev, time) == (0.37, 1.0):
            assert edits == ["update_materials", "update_lights"] and pt.bvh_build_ms() != ms     # transmission 0 -> 0.5: rebuilt
        if (prev, time) == (1.0, 1.6):
            assert "set_node_visibility" in edits and pt.bvh_build_ms() != ms
        locals_, weights = _feed(pt, scn, tasks, time, first=k == 0)
        got = _snapshot(pt, res)
        ptB, resB = _attach(_clone(scn), std_env, builder)
        _feed(ptB, scn, tasks, time, first=True)
        want = _snapshot(ptB, resB)
        ptB.onDetach()
        for key in ("img", "ids", "depth"):
            assert np.array_equal(got[key].view(np.uint32), want[key].view(np.uint32)), (builder, time, key)
        assert got["stats"] == want["stats"], (builder, time, got["stats"], want["stats"])
        if time in ORACLE_TIMES and prev != time:
            e = rel_rmse(got["img"], _oracle_image(oracle_mod, scn, tasks, locals_, weights, std_env))
            print(builder, time, "rel RMSE", e)
            assert np.isfinite(got["img"]).all() and e <= 1e-3, (builder, time, e)
        prev = time
    pt.onDetach()
