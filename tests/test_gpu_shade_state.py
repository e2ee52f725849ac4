"""-m gpu: the device's hit fetch, getHitState and evaluateMaterial (k_shade_state through b200pt_shade_state, the frame's
walk and the frame's shade variant) against the float64 restatement of tests/hitref.py and against the CPU oracle.

The scenes and assertion groups 1-2 are those of test_shade_state.py.  Group 3, device against oracle: bit for bit on every
field, except the scatter coefficient (logf) and, on records with a texture gradient, the fields built from texture fetches
(a log2f ulp moves a trilinear weight, as test_gpu_textures.py allows): those within 1e-6 relative of the oracle's.

Geometry the device rewrote: the device reads the shade records gathered at scene build through shadeIdx[slot], and
re-gathered by k_regather_shade after an animation; the oracle and hitref read the primitive arrays.  So the animated scene
at a bent pose (reference arrays from oracle/animation.apply), the node hierarchy after update_node_matrices (its mirrored
chain included), an in-place material edit and a material-variant switch are run as well, every scene under both builders.

Variant gating: a scene without extension features runs k_shade<0>, a clearcoat-only scene k_shade<FEAT_LEAN>.  There a gated
instantiation may leave a field as the ungated reference would not; each such field is named in GATED with the record
condition that makes it unreachable, the gated scenes make every one of them differ, and any other difference fails."""
import copy

import numpy as np
import pytest

import hitref
from test_shade_state import (BRANCH_SIDES, TEXTURED, add_readback, aimed_rays, attribute_zoo, check_independent, compare_reference,
                              scenes, stored_levels, sweep_records)
from vk_gltf_renderer_b200 import shade_io, synth
from vk_gltf_renderer_b200.scene import Camera, Scene

pytestmark = pytest.mark.gpu

# field -> record condition under which a gated variant may differ from the reference: the lobe that reads it has weight 0
# (shade.cuh: evaluateMaterial skips the texture, or the field, when the variant leaves the feature out)
_zero = lambda name: (lambda out: np.all(np.atleast_2d(shade_io.field(out, name).T).T == 0, axis=1))
GATED = {
    "sheenRoughness": _zero("sheenColor"),                       # sheen lobe weight 0
    "iridescenceThickness": _zero("iridescence"),                # no thin film
    "clearcoatRoughness": _zero("clearcoat"),                    # clearcoat lobe weight 0
    "Nc": _zero("clearcoat"),
    "diffuseTransmissionColor": _zero("diffuseTransmissionFactor"),  # diffuse-transmission lobe weight 0
    "dispersion": _zero("transmission"),                         # no specular transmission
}
# which gated fields each gated scene makes differ
GATED_SEEN = {False: set(GATED), True: set(GATED) - {"clearcoatRoughness", "Nc"}}


def _device(scene, builder=0):
    from vk_gltf_renderer_b200.renderer import PathTracer, Resources
    pt = PathTracer(0)
    res = Resources(scene=scene, camera=scene.camera or Camera(), size=(8, 8))
    pt.onAttach(res)
    if builder:
        pt.set_bvh_builder(builder)
        pt.onSceneInvalidated(res)
    return pt, res


def _clone(scn):
    return synth.scene_from_state(copy.deepcopy(synth.scene_state(scn)))


def _calls(pt):
    import torch

    def lookup(records):
        records = np.ascontiguousarray(records, np.float32).reshape(-1, 8)
        d_in = torch.from_numpy(records).cuda()
        d_out = torch.empty((len(records), 4), dtype=torch.float32, device="cuda")
        pt.texture_lookup(d_in.data_ptr(), len(records), d_out.data_ptr())
        pt.synchronize()
        return d_out.cpu().numpy()

    def shade(records, seeds):
        d_in = torch.from_numpy(np.ascontiguousarray(records, np.float32)).cuda()
        d_out = torch.full((len(records), shade_io.OUT_FLOATS), np.nan, dtype=torch.float32, device="cuda")
        d_seeds = torch.from_numpy(seeds.view(np.int32).copy()).cuda()
        pt.shade_state(d_in.data_ptr(), len(records), d_out.data_ptr(), d_seeds.data_ptr())
        pt.synchronize()
        seeds[:] = d_seeds.cpu().numpy().view(np.uint32)
        return d_out.cpu().numpy()
    return lookup, shade


def compare_oracle(dev, ora, rec_in, tag):
    """group 3; returns the largest deviation per field"""
    hit = shade_io.field(ora, "t") < shade_io.MISS_T
    assert np.array_equal(dev[:, :6], ora[:, :6]), (tag, "hits differ")
    grad = hit & (shade_io.field(ora, "texGrad") > 0)
    worst = {}
    for name in shade_io.FIELDS:
        a, b = shade_io.field(dev, name), shade_io.field(ora, name)
        same = (a == b) if a.ndim == 1 else np.all(a == b, axis=1)
        loose = grad if name in TEXTURED else np.zeros_like(grad)
        if name == "scatterCoefficient":
            loose = hit
        d = np.abs(a.astype(np.float64) - b)
        d = d if d.ndim == 1 else d.max(1)
        close = d <= 1e-6 * (1.0 + np.abs(b if b.ndim == 1 else b.max(1)))
        bad = np.flatnonzero(~same & ~(loose & close))
        assert len(bad) == 0, (tag, name, len(bad), bad[:4], a[bad[:4]], b[bad[:4]])
        worst[name] = float(d.max())
    return worst


def _run(oracle_mod, tag, pt, scn, ims, per_node, cone, seed, stats, gated=False):
    """the records of one handle `pt` against the oracle and hitref on `scn`, the description of what the handle holds now"""
    lookup, shade = _calls(pt)
    o = oracle_mod.Oracle()
    o.set_scene(scn)
    levels = stored_levels(lookup, ims)
    ora_levels = stored_levels(o.texture_lookup, ims)
    assert all(np.array_equal(a, b) for k in levels for a, b in zip(levels[k], ora_levels[k])), tag
    rays = aimed_rays(scn, per_node, seed=seed)
    rec = sweep_records(rays, seed=seed + 100, cone=cone)
    seeds = np.arange(len(rec), dtype=np.uint32) * 2654435761
    s_dev, s_ora = seeds.copy(), seeds.copy()
    dev = shade(rec, s_dev)
    ora = o.shade_state(rec, s_ora)
    assert np.array_equal(s_dev, s_ora), tag
    check_independent(scn, rec, dev, tag)
    sref = hitref.SceneRef(scn, levels)
    fields = [k for k in shade_io.FIELDS if shade_io.FIELDS[k][0] >= 6 and not (gated and k in GATED)]
    compare_reference(sref, rec, dev, tag, fields=fields, stats=stats)
    if gated:
        # each gated field: equal to the oracle's (ungated) value, or unreachable in that record
        hit = shade_io.field(dev, "t") < shade_io.MISS_T
        for name, unreachable in GATED.items():
            # beyond the log2f ulp a textured field may carry (group 3)
            d = np.abs(shade_io.field(dev, name).astype(np.float64) - shade_io.field(ora, name))
            d = d if d.ndim == 1 else d.max(1)
            differs = hit & (d > 1e-6 * (1.0 + np.abs(shade_io.field(ora, name)).reshape(len(d), -1).max(1)))
            assert (unreachable(dev)[differs]).all(), (tag, name)
            stats.setdefault("gated", {})[name] = stats.get("gated", {}).get(name, 0) + int(differs.sum())
        dev = dev.copy()
        for name in GATED:
            a, w = shade_io.FIELDS[name]
            dev[:, a:a + w] = ora[:, a:a + w]
    w = compare_oracle(dev, ora, rec, tag)
    for k, v in w.items():
        stats.setdefault("vs_oracle", {})[k] = max(stats.get("vs_oracle", {}).get(k, 0.0), v)


def _gated_scene(clearcoat):
    """a plain scene (k_shade<0>) or a clearcoat-only one (k_shade<FEAT_LEAN>) whose material binds the textures of features
    it leaves at factor 0 (sheen roughness, iridescence thickness, clearcoat roughness and normal, diffuse-transmission
    colour), has a dispersion without transmission, and a normal map"""
    rng = np.random.default_rng(5)
    scn = Scene()
    base, mr, nm = synth.make_texture_set(32, rng, (0.7, 0.7, 0.7))
    tb, tm, tn = scn.add_texture(base, srgb=True), scn.add_texture(mr), scn.add_texture(nm)
    ts = scn.add_texture(synth._u8(0.2 + 0.8 * synth.value_noise(32, 4, rng, 4)))      # varied alpha: the sheen roughness
    # textures bound to features whose factor is 0 (which keeps them out of the variant), and a dispersion without transmission
    m = scn.add_material(pbrBaseColorFactor=[1, 1, 1, 1], pbrRoughnessFactor=0.7, pbrMetallicFactor=0.3, pbrBaseColorTexture=scn.add_texture_info(tb),
                         pbrMetallicRoughnessTexture=scn.add_texture_info(tm), normalTexture=scn.add_texture_info(tn),
                         sheenRoughnessFactor=0.5, sheenRoughnessTexture=scn.add_texture_info(ts),
                         iridescenceThicknessMinimum=100.0, iridescenceThicknessMaximum=400.0, iridescenceThicknessTexture=scn.add_texture_info(ts),
                         clearcoatFactor=0.7 if clearcoat else 0.0, clearcoatRoughness=0.4, clearcoatRoughnessTexture=scn.add_texture_info(ts),
                         clearcoatNormalTexture=scn.add_texture_info(tn), diffuseTransmissionColor=[0.8, 0.7, 0.6],
                         diffuseTransmissionColorTexture=scn.add_texture_info(ts), dispersion=0.3)
    sp = synth._sphere(0.0, 0.0, 0.0, 0.8, n=16)
    scn.add_node(scn.add_primitive(sp[0], sp[4], normals=sp[1], uv0=sp[2], tangents=sp[3]), m)
    M = np.diag([1.3, 0.6, 1.0, 1.0])
    M[0, 3] = 2.0
    scn.add_node(scn.add_primitive(sp[0], sp[4], normals=sp[1], uv0=sp[2]), m, M)
    cam = Camera()
    cam.eye = np.array([0.0, 0.0, 5.0], np.float32)
    scn.camera = cam
    return scn


def _report(stats, what):
    print(f"{what}: {stats['records']} hits, {stats['near']} within a branch margin; largest deviation per field (hitref, oracle)")
    for k in sorted(stats["worst"]):
        print(f"  {k:28s} {stats['worst'][k]:.3e}   {stats['vs_oracle'].get(k, 0.0):.3e}")


@pytest.mark.parametrize("builder", [0, 1])
def test_device_hit_state_matches_float64_reference_and_oracle(oracle_mod, builder):
    stats = {}
    for k, (tag, scn, per_node, cone) in enumerate(scenes()):
        ims = add_readback(scn)
        pt, _ = _device(scn, builder)
        _run(oracle_mod, tag, pt, scn, ims, per_node, cone, 300 + k, stats)
    for b in BRANCH_SIDES:
        assert stats["taken"].get(b) == {False, True}, (b, stats["taken"].get(b))
    _report(stats, f"builder {builder}")


@pytest.mark.parametrize("builder", [0, 1])
def test_device_hit_state_after_animation(oracle_mod, builder):
    """morph + skin at a bent pose: the device re-gathers the shade records of the posed primitives (k_regather_shade) and
    refits; the reference reads the arrays oracle/animation.apply poses"""
    from oracle import animation as A
    scn, morphs, skins, pose = synth.synth_animated()
    ims = add_readback(scn)
    rest = _clone(scn)
    pt, _ = _device(scn, builder)
    pt.set_animation(morphs, skins)
    stats = {}
    for k in (1, 2):
        mw, jm, nm = pose(k)
        pt.animate(mw, jm, nm)
        ref = _clone(rest)
        A.apply(ref, morphs, skins, mw, jm, nm)
        _run(oracle_mod, f"animated pose {k}", pt, ref, ims, 120, (2e-3, 4e-3), 600 + k, stats)
    _report(stats, f"animated, builder {builder}")


@pytest.mark.parametrize("builder", [0, 1])
def test_device_hit_state_after_node_matrix_updates(oracle_mod, builder):
    """b200pt_update_node_matrices rewrites the render nodes (a mirrored chain among them) and refits; the reference reads the
    render nodes oracle/animation.py computes"""
    from oracle import animation as A
    from vk_gltf_renderer_b200.animation import topo_levels
    scn, parents, mappings, inst, pose = synth.synth_hierarchy()
    ims = add_readback(scn)
    glm = lambda ms: np.ascontiguousarray(np.asarray(ms, np.float64).transpose(0, 2, 1).astype(np.float32))
    pt, _ = _device(scn, builder)
    pt.set_node_hierarchy(parents, mappings, glm(inst))
    order, offsets = topo_levels(parents)
    stats = {}
    for k in (1, 2):
        loc = glm(pose(k))
        pt.update_node_matrices(loc)
        o2w, w2o = A.render_nodes(A.propagate(loc, parents, order, offsets), mappings, glm(inst))
        assert (np.linalg.det(o2w[:, :3, :3]) < 0).any()      # the mirrored chain
        ref = _clone(scn)
        for i, rn in enumerate(ref.render_nodes):
            rn["objectToWorld"], rn["worldToObject"] = o2w[i].reshape(-1).copy(), w2o[i].reshape(-1).copy()
        _run(oracle_mod, f"hierarchy pose {k}", pt, ref, ims, 160, (2e-3, 4e-3), 700 + k, stats)
    _report(stats, f"hierarchy, builder {builder}")


@pytest.mark.parametrize("builder", [0, 1])
def test_device_hit_state_after_material_edit_and_variant_switch(oracle_mod, builder):
    """an in-place b200pt_update_materials (factors, normal scale, a texture slot rebound) and a b200pt_update_node_materials
    variant switch: the records must read the edited tables"""
    scn = synth.synth_material_zoo()
    ims = add_readback(scn)
    pt, res = _device(scn, builder)
    stats = {}
    m = scn.materials[3]
    m.pbrBaseColorFactor[0], m.pbrRoughnessFactor, m.normalTextureScale = 0.9, 0.15, -1.7
    scn.materials[4].clearcoatFactor = 0.4
    scn.materials[0].sheenRoughnessTexture = scn.materials[4].clearcoatRoughnessTexture
    pt.update_materials(res)
    _run(oracle_mod, "material edit", pt, _clone(scn), ims, 64, (2e-3, 4e-3), 800, stats)
    nodes = scn.render_nodes
    nodes[1]["materialID"], nodes[2]["materialID"], nodes[7]["materialID"] = nodes[2]["materialID"], nodes[7]["materialID"], nodes[1]["materialID"]
    pt.update_node_materials(res)
    _run(oracle_mod, "variant switch", pt, _clone(scn), ims, 64, (2e-3, 4e-3), 801, stats)
    _report(stats, f"edits, builder {builder}")


@pytest.mark.parametrize("clearcoat", [False, True], ids=["k_shade0", "k_shade_lean"])
def test_device_gated_variants_differ_only_where_unreachable(oracle_mod, clearcoat):
    stats = {}
    scn = _gated_scene(clearcoat)
    ims = add_readback(scn)
    pt, _ = _device(scn)
    _run(oracle_mod, "lean" if clearcoat else "plain", pt, scn, ims, 400, (2e-3, 4e-3), 500, stats, gated=True)
    print("gated fields that differed (unreachable):", stats.get("gated"))
    seen = {k for k, v in stats["gated"].items() if v > 0}
    assert seen == GATED_SEEN[clearcoat], seen      # every gate the scene binds is exercised


def test_shade_state_refuses_without_scene_or_buffers():
    import torch
    from vk_gltf_renderer_b200.renderer import B200PTError, PathTracer
    pt = PathTracer(0)
    d = torch.zeros(16, device="cuda")
    with pytest.raises(B200PTError):
        pt.shade_state(d.data_ptr(), 1, d.data_ptr())
    scn = attribute_zoo()
    pt2, _ = _device(scn)
    with pytest.raises(B200PTError):
        pt2.shade_state(0, 1, d.data_ptr())
