"""-m gpu scene edits (b200pt_update_materials / update_node_materials / update_lights / set_node_visibility, the steps of
GltfRenderer::updateSceneChanges): after any sequence of edits a handle renders exactly what a fresh handle renders when
b200pt_set_scene gets the edited description -- accumulation RGB and .w, selection ids and NDC depth, the stats counters and
the ray-level API's hits, seeds and transmission, bit for bit, with the same BVH builder on both handles."""
import copy

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SIZE = (96, 72)
FRAMES = 3
STATS = ("closestRays", "shadowRays", "shadedHits", "pathsStarted")


def _clone(scn):
    from vk_gltf_renderer_b200 import synth
    c = synth.scene_from_state(copy.deepcopy(synth.scene_state(scn)))
    c.micromaps, c.prim_omms = scn.micromaps, scn.prim_omms
    return c


def _attach(scn, env, builder=0, depth=5):
    from vk_gltf_renderer_b200.renderer import PathTracer, Resources
    res = Resources(scene=scn, hdr_rgb=env, camera=scn.camera, size=SIZE)
    pt = PathTracer(0)
    pt.ptMaxDepth = depth
    pt.onAttach(res)
    if builder:
        pt.set_bvh_builder(builder)
        pt.onSceneInvalidated(res)
    return pt, res


def _render(pt, res, frames=FRAMES):
    for f in range(frames):
        res.frameCount = f
        pt.onRender(None, res)
    pt.flush()
    pt.synchronize()


def _snapshot(pt, res, rays=None):
    """what the handle renders now: image, selection, counters, and the ray-level answers"""
    import torch
    from gpu_util import random_rays, to_dev
    pt.reset_stats()
    _render(pt, res)
    out = dict(img=pt.read_accum())
    out["ids"], out["depth"] = pt.read_selection()
    st = pt.stats()
    out["stats"] = [st[k] for k in STATS]
    lo, hi = res.scene.bounds()
    r = random_rays(30000, lo, hi, seed=7)
    seeds = (torch.arange(len(r), dtype=torch.int64, device="cuda") * 2654435761 % (1 << 31)).to(torch.int32)
    s0 = seeds.clone()
    hits = torch.empty((len(r), 6), dtype=torch.float32, device="cuda")
    pt.trace_closest(to_dev(r).data_ptr(), len(r), hits.data_ptr(), s0.data_ptr())
    r[:, 7] = float(np.linalg.norm(hi - lo))
    s1 = seeds.clone()
    trans = torch.empty((len(r), 3), dtype=torch.float32, device="cuda")
    pt.trace_shadow(to_dev(r).data_ptr(), len(r), trans.data_ptr(), s1.data_ptr())
    pt.synchronize()
    out["hits"], out["trans"], out["seeds"] = hits.cpu().numpy(), trans.cpu().numpy(), np.stack([s0.cpu().numpy(), s1.cpu().numpy()])
    return out


def _assert_same(a, b, tag, stats=True):
    for k in ("img", "ids", "depth", "hits", "trans", "seeds"):
        assert np.array_equal(np.asarray(a[k]).view(np.uint32), np.asarray(b[k]).view(np.uint32)), (tag, k)
    if stats:
        assert a["stats"] == b["stats"], (tag, a["stats"], b["stats"])


def _fresh(scn, env, builder=0, depth=5):
    pt, res = _attach(_clone(scn), env, builder, depth)
    s = _snapshot(pt, res)
    pt.onDetach()
    return s


def _edit_and_compare(pt, res, env, edit, push, tag, builder=0):
    """apply `edit` to the scene of (pt, res), push it with pt.<push>(res), compare with a fresh handle"""
    edit(res.scene)
    for p in push:
        getattr(pt, p)(res)
    _assert_same(_snapshot(pt, res), _fresh(res.scene, env, builder), tag)


# ---- 1. material values (in place) -----------------------------------------------------------------------------------------

def test_material_values(std_env):
    from vk_gltf_renderer_b200 import synth
    scn = synth.synth_material_zoo()
    pt, res = _attach(scn, std_env)
    _render(pt, res)
    M = scn.materials
    opaque = [i for i, m in enumerate(M) if m.alphaMode == 0 and m.transmissionFactor == 0 and m.diffuseTransmissionFactor == 0]
    assert len(opaque) >= 3

    def colour(s):
        s.materials[opaque[0]].pbrBaseColorFactor[:] = [0.2, 0.9, 0.3, 1.0]

    def roughness(s):
        s.materials[opaque[1]].pbrRoughnessFactor = 0.05

    def emission(s):
        s.materials[opaque[2]].emissiveFactor[:] = [3.0, 0.5, 0.5]

    def double_sided(s):
        s.materials[opaque[1]].doubleSided = 1 - s.materials[opaque[1]].doubleSided

    def new_texture_table(s):
        ti = s.add_texture_info(0, 1, (2, 0, 0, 2, 0.5, 0.25))
        s.materials[opaque[0]].pbrBaseColorTexture = ti
    for f in (colour, roughness, emission, double_sided, new_texture_table):
        _edit_and_compare(pt, res, std_env, f, ["update_materials"], f.__name__)
    pt.onDetach()


def test_sheen_turned_on_flips_the_lean_shade_variant(std_env):
    from vk_gltf_renderer_b200 import synth
    scn = synth.synth_lit()   # no sheen, no transmission: the lean shade variant
    pt, res = _attach(scn, std_env)
    _render(pt, res)

    def sheen(s):
        s.materials[1].sheenColorFactor[:] = [0.8, 0.2, 0.9]
        s.materials[1].sheenRoughnessFactor = 0.4

    def sheen_off(s):
        s.materials[1].sheenColorFactor[:] = [0.0, 0.0, 0.0]
    _edit_and_compare(pt, res, std_env, sheen, ["update_materials"], "sheen on")
    _edit_and_compare(pt, res, std_env, sheen_off, ["update_materials"], "sheen off")
    pt.onDetach()


# ---- 2. alpha classes (in place and rebuilt) --------------------------------------------------------------------------------

def _alpha_steps():
    def cutoff(s):
        s.materials[0].alphaCutoff = 0.3

    def opaque_to_mask(s):    # the floor joins the any-hit geometry
        s.materials[1].alphaMode = 1
        s.materials[1].alphaCutoff = 0.5

    def mask_to_blend(s):
        s.materials[0].alphaMode = 2

    def mask_to_opaque(s):
        s.materials[1].alphaMode = 0

    def last_non_opaque_made_opaque(s):
        s.materials[0].alphaMode = 0

    def transmission_on(s):
        s.materials[1].transmissionFactor = 0.8
        s.materials[1].thicknessFactor = 0.0
    return [cutoff, opaque_to_mask, mask_to_blend, mask_to_opaque, last_non_opaque_made_opaque, transmission_on]


@pytest.mark.parametrize("builder", [0, 1])
def test_alpha_classes(std_env, builder):
    from vk_gltf_renderer_b200 import synth
    scn = synth.synth_layers(layers=6)
    pt, res = _attach(scn, std_env, builder)
    _render(pt, res)
    for f in _alpha_steps():
        _edit_and_compare(pt, res, std_env, f, ["update_materials"], f"builder {builder}: {f.__name__}", builder)
    pt.onDetach()


def test_alpha_classes_with_sampler_layers(std_env):
    from vk_gltf_renderer_b200 import synth
    scn = synth.sampler_layers()
    pt, res = _attach(scn, std_env)
    _render(pt, res)
    ground = len(scn.materials) - 1

    def cutoffs(s):
        for m in s.materials[:ground]:
            m.alphaCutoff = 0.35

    def ground_masked(s):
        s.materials[ground].alphaMode = 1

    def layers_opaque(s):
        for m in s.materials[:ground]:
            m.alphaMode = 0
    for f in (cutoffs, ground_masked, layers_opaque):
        _edit_and_compare(pt, res, std_env, f, ["update_materials"], f.__name__)
    pt.onDetach()


def test_alpha_classes_with_micromaps(std_env):
    from vk_gltf_renderer_b200 import omm, synth
    scn = synth.synth_layers(layers=6)
    omm.bake_opacity_micromaps(scn, level=3)
    pt, res = _attach(scn, std_env)
    _render(pt, res)

    def cutoff(s):   # in place: the links stay
        s.materials[0].alphaCutoff = 0.5

    def opaque(s):   # no non-opaque triangle left: no links
        s.materials[0].alphaMode = 0

    def mask_again(s):  # linked again
        s.materials[0].alphaMode = 1
    for f in (cutoff, opaque, mask_again):
        _edit_and_compare(pt, res, std_env, f, ["update_materials"], f.__name__)
    pt.onDetach()


# ---- 3. variants -------------------------------------------------------------------------------------------------------------

def test_variant_swap_and_back(std_env):
    from vk_gltf_renderer_b200 import synth
    scn = synth.synth_lit()
    pt, res = _attach(scn, std_env)
    _render(pt, res)
    a, b = scn.render_nodes[1]["materialID"], scn.render_nodes[2]["materialID"]

    def swap(s):
        s.render_nodes[1]["materialID"], s.render_nodes[2]["materialID"] = b, a

    def back(s):
        s.render_nodes[1]["materialID"], s.render_nodes[2]["materialID"] = a, b
    _edit_and_compare(pt, res, std_env, swap, ["update_node_materials"], "swap")
    _edit_and_compare(pt, res, std_env, back, ["update_node_materials"], "back")
    pt.onDetach()


def test_variant_switch_survives_node_matrix_updates(std_env):
    """with a node hierarchy, the switched ids must also reach the mappings b200pt_update_node_matrices rewrites the nodes from"""
    from vk_gltf_renderer_b200 import synth
    scn, parents, mappings, inst, pose = synth.synth_hierarchy()
    glm = lambda L: np.ascontiguousarray(np.transpose(L, (0, 2, 1)), np.float32)
    pt, res = _attach(scn, std_env)
    pt.set_node_hierarchy(parents, mappings, glm(inst))
    pt.update_node_matrices(glm(pose(1)))
    _render(pt, res)
    scn.render_nodes[1]["materialID"], scn.render_nodes[3]["materialID"] = scn.render_nodes[3]["materialID"], scn.render_nodes[1]["materialID"]
    pt.update_node_materials(res)
    pt.update_node_matrices(glm(pose(2)))
    got = _snapshot(pt, res)
    ptB, resB = _attach(_clone(scn), std_env)
    ptB.set_node_hierarchy(parents, [(g, rn["materialID"], p) for (g, _, p), rn in zip(mappings, scn.render_nodes)], glm(inst))
    ptB.update_node_matrices(glm(pose(1)))
    ptB.update_node_matrices(glm(pose(2)))
    _assert_same(got, _snapshot(ptB, resB), "hierarchy")
    pt.onDetach()
    ptB.onDetach()


# ---- 4. visibility -----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("builder", [0, 1])
def test_visibility(std_env, builder):
    from vk_gltf_renderer_b200 import synth
    scn = synth.synth_layers(layers=6)
    mirror = np.diag([-1.0, 1.0, 1.0, 1.0])
    mirror[:3, 3] = [0.4, 0.0, -1.2]
    scn.add_node(scn.render_nodes[2]["renderPrimID"], scn.render_nodes[2]["materialID"], mirror)   # an instanced, mirrored copy
    pt, res = _attach(scn, std_env, builder)
    _render(pt, res)
    n = len(scn.render_nodes)
    non_opaque = [i for i in range(n) if scn.materials[max(0, scn.render_nodes[i]["materialID"])].alphaMode != 0]

    def hide(idx):
        def f(s):
            for i in idx:
                s.render_nodes[i]["visible"] = False
        return f

    def show_all(s):
        for rn in s.render_nodes:
            rn["visible"] = True
    for tag, f in (("one node", hide([1])), ("mirrored instance", hide([n - 1])), ("all non-opaque", hide(non_opaque)), ("all shown", show_all)):
        _edit_and_compare(pt, res, std_env, f, ["set_node_visibility"], f"builder {builder}: {tag}", builder)
    pt.onDetach()


def test_visibility_keeps_an_animated_pose(std_env):
    """A is posed, then a node is hidden (its trees are rebuilt over the posed vertices); B is set up hidden, then posed.  The trees
    are built over different poses, so they differ in shape and the traversal counters may differ; what the rays see does not."""
    from vk_gltf_renderer_b200 import synth
    scn, morphs, skins, pose = synth.synth_animated()
    mw, jm, nm = pose(1)
    pt, res = _attach(scn, std_env)
    pt.set_animation(morphs, skins)
    pt.animate(mw, jm, nm)
    _render(pt, res)
    scn.render_nodes[0]["visible"] = False
    pt.set_node_visibility(res)
    got = _snapshot(pt, res)
    ptB, resB = _attach(_clone(scn), std_env)
    ptB.set_animation(morphs, skins)
    ptB.animate(mw, jm, nm)
    _assert_same(got, _snapshot(ptB, resB), "posed, then hidden", stats=False)
    pt.onDetach()
    ptB.onDetach()


# ---- 5. lights ---------------------------------------------------------------------------------------------------------------

def test_lights(std_env):
    from vk_gltf_renderer_b200 import synth
    scn = synth.synth_lit()
    pt, res = _attach(scn, std_env)
    _render(pt, res)
    five = list(scn.lights)

    def edit_values(s):
        s.lights[0].color[:] = [0.2, 1.0, 0.4]
        s.lights[1].intensity = 30.0
        s.lights[0].position[:] = [1.0, 2.5, -0.5]
        s.lights[2].outerAngle = 0.8
        s.lights[2].innerAngle = 0.1

    def one(s):
        s.lights = five[:1]

    def none(s):
        s.lights = []

    def two(s):
        s.lights = five[2:4]
    for f in (edit_values, one, none, two):
        _edit_and_compare(pt, res, std_env, f, ["update_lights"], f.__name__)
    pt.onDetach()


# ---- 6. scheduling -----------------------------------------------------------------------------------------------------------

def test_edit_with_a_partial_frame_batch(std_env):
    """an edit arriving while 2 of a batch of 3 frames are pending (4 frames in flight) renders them with the old scene first"""
    from vk_gltf_renderer_b200 import synth

    def run(batch, lanes):
        scn = synth.synth_layers(layers=6)
        pt, res = _attach(scn, std_env)
        pt.set_frames_in_flight(lanes)
        pt.set_frame_batch(batch)
        for f in range(5):
            res.frameCount = f
            pt.onRender(None, res)
        scn.materials[0].alphaMode = 2
        scn.materials[1].pbrBaseColorFactor[:] = [0.9, 0.3, 0.3, 1.0]
        pt.update_materials(res)
        for f in range(5, 9):
            res.frameCount = f
            pt.onRender(None, res)
        pt.flush()
        pt.synchronize()
        img = pt.read_accum()
        pt.onDetach()
        return img
    assert np.array_equal(run(3, 4).view(np.uint32), run(1, 1).view(np.uint32))


# ---- 7. refusals -------------------------------------------------------------------------------------------------------------

def test_refused_edits_leave_the_scene_as_it_was(std_env):
    import ctypes as C
    from vk_gltf_renderer_b200 import abi, synth
    from vk_gltf_renderer_b200.renderer import B200PTError, Resources
    scn = synth.synth_layers(layers=4)
    scn.materials[0].alphaMode = 0   # every layer opaque: micromaps are not linked, so one too short for its primitive is accepted
    tri = np.zeros(1, abi.MICROMAP_TRIANGLE_DTYPE)
    tri["format"] = abi.OMM_FORMAT_4_STATE
    scn.micromaps = [dict(data=np.zeros(4, np.uint8), triangles=tri)]
    scn.prim_omms = [dict(renderPrimID=scn.render_nodes[0]["renderPrimID"], micromap=0, baseTriangle=0, indices=None)]
    pt, res = _attach(scn, std_env)
    before = _snapshot(pt, res)
    L, h = pt._L, pt._h
    n = len(scn.render_nodes)
    mats = (abi.ShadeMaterial * len(scn.materials))(*scn.materials)
    tis = (abi.TextureInfo * len(scn.texture_infos))(*scn.texture_infos)
    assert L.b200pt_update_materials(h, mats, len(scn.materials) - 1, tis, len(scn.texture_infos)) == -1   # material count
    ids = np.zeros(n + 1, np.int32)
    ids[0] = len(scn.materials)
    assert L.b200pt_update_node_materials(h, ids.ctypes.data_as(C.POINTER(C.c_int32)), n) == -1       # material id >= count
    ids[0] = 0
    assert L.b200pt_update_node_materials(h, ids.ctypes.data_as(C.POINTER(C.c_int32)), n + 1) == -1   # node count
    vis = np.ones(n + 1, np.uint8)
    assert L.b200pt_set_node_visibility(h, vis.ctypes.data_as(C.POINTER(C.c_uint8)), n + 1) == -1     # node count

    def refused(edit, rc):
        s = _clone(scn)
        edit(s)
        with pytest.raises(B200PTError) as e:
            pt.update_materials(Resources(scene=s))
        assert f"({rc})" in str(e.value), str(e.value)

    refused(lambda s: setattr(s.materials[0], "pbrBaseColorTexture", len(s.texture_infos)), -1)   # texture slot beyond the table
    refused(lambda s: setattr(s.materials[0], "retroreflectionFactor", 0.5), -4)                  # B200PT_E_UNSUPPORTED
    refused(lambda s: setattr(s.materials[0], "alphaMode", 1), -1)   # non-opaque now: the micromap does not cover the primitive
    _assert_same(_snapshot(pt, res), before, "after the refusals")
    pt.onDetach()
