"""-m gpu parity for the rows round 1 left without a GPU test: punctual lights (FEAT_LIGHTS), every KHR_materials_* extension
WITH its textures (FEAT_ALL), and the device-side error flag of the tree walks."""
import numpy as np
import pytest

from conftest import rel_rmse

pytestmark = pytest.mark.gpu


def _oracle(oracle_mod, scene, env):
    o = oracle_mod.Oracle()
    o.set_scene(scene)
    o.set_environment(env)
    return o


def _gpu_render(scene, env, w, h, frames, **kw):
    from vk_gltf_renderer_b200.renderer import render_headless, Resources
    res = Resources(scene=scene, hdr_rgb=env, camera=scene.camera, size=(w, h))
    return render_headless(res, frames, **kw)


def test_render_parity_punctual_lights(std_env, oracle_mod):
    """Point (radius 0 and > 0), spot with range, directional with and without angular size: sampleLights' light branch,
    singleLightContribution, light / environment technique MIS (pathtrace_functions.h.slang:396-412; GltfLight as
    src/gltf_scene_vk.cpp:1354-1394 fills it).  Stream-replicated: rel RMSE <= 1e-3, identical ray budgets."""
    from vk_gltf_renderer_b200 import synth
    scn = synth.synth_lit()
    assert len(scn.lights) == 5
    o = _oracle(oracle_mod, scn, std_env)
    ref = oracle_mod.render(o, scn.camera, 192, 128, 8, max_depth=6)
    pt, img = _gpu_render(scn, std_env, 192, 128, 8, ptMaxDepth=6)
    assert np.isfinite(img).all()
    e = rel_rmse(img, ref)
    print("lights rel RMSE", e)
    assert e <= 1e-3
    # .w is the running mean of the primary hit's solid flag -- scaled by the firefly clamp wherever a sample's luminance
    # exceeds the threshold (gltf_pathtrace.slang:533-538: the clamp multiplies all four channels), which the bright
    # punctual lights trigger, so it is compared to rounding rather than bit for bit
    assert np.allclose(img[..., 3], ref[..., 3], rtol=1e-5, atol=1e-6)
    st, so = pt.stats(), o.stats()
    assert st["closestRays"] == so["closestRays"] and st["shadowRays"] == so["shadowRays"]
    # the lights matter: the same scene without them is clearly darker
    scn.lights = []
    _, dark = _gpu_render(scn, std_env, 192, 128, 2, ptMaxDepth=6)
    assert dark[..., :3].mean() < 0.8 * img[..., :3].mean()


def test_render_parity_material_zoo_all_extensions_textured(std_env, oracle_mod):
    """Sheen, iridescence (+ thickness texture on TEXCOORD_1), anisotropy (+ direction texture under KHR_texture_transform),
    specular / specular colour, clearcoat (+ roughness + normal textures), transmission + thickness textures with volume
    attenuation, diffuse transmission (+ colour texture), pbrSpecularGlossiness with both textures, emissive texture, BLEND
    alpha, vertex colours: evaluateMaterial + bsdfEvaluate / bsdfSample of the FEAT_ALL shade variant against the oracle,
    stream-replicated, rel RMSE <= 1e-3 (gltf_material_eval.h.slang:168-457)."""
    from vk_gltf_renderer_b200 import synth
    scn = synth.synth_material_zoo()
    o = _oracle(oracle_mod, scn, std_env)
    ref = oracle_mod.render(o, scn.camera, 240, 160, 8, max_depth=8)
    pt, img = _gpu_render(scn, std_env, 240, 160, 8, ptMaxDepth=8)
    assert np.isfinite(img).all()
    e = rel_rmse(img, ref)
    print("material zoo rel RMSE", e)
    assert e <= 1e-3
    st, so = pt.stats(), o.stats()
    assert abs(st["closestRays"] / so["closestRays"] - 1.0) <= 1e-3


def test_render_parity_dispersion(std_env, oracle_mod):
    """KHR_materials_dispersion (BASELINE config 4's feature; SynthGlass stand-in with dispersion 20, SURVEY.md section 8d):
    one colour channel per refraction event with the per-channel IOR of gltf_raster.slang:204-208.  Stream-replicated
    parity with the oracle, and the effect is there: the image differs from the dispersion-free render in chroma only."""
    from vk_gltf_renderer_b200 import synth
    scn = synth.synth_glass(n=48, dispersion=20.0)
    o = _oracle(oracle_mod, scn, std_env)
    ref = oracle_mod.render(o, scn.camera, 128, 128, 8, max_depth=12)
    pt, img = _gpu_render(scn, std_env, 128, 128, 8, ptMaxDepth=12)
    assert np.isfinite(img).all()
    e = rel_rmse(img, ref)
    print("dispersion rel RMSE", e)
    assert e <= 1e-3
    _, plain = _gpu_render(synth.synth_glass(n=48), std_env, 128, 128, 8, ptMaxDepth=12)
    assert rel_rmse(img, plain) > 0.05
    sat = lambda a: float((a[..., :3].max(-1) - a[..., :3].min(-1)).mean())
    assert sat(img) > 1.05 * sat(plain)


def test_retroreflection_is_rejected_not_ignored(box_scene, std_env):
    import copy
    from vk_gltf_renderer_b200 import synth
    from vk_gltf_renderer_b200.renderer import B200PTError, PathTracer, Resources
    scn = synth.scene_from_state(copy.deepcopy(synth.scene_state(box_scene)))
    scn.materials[0].retroreflectionFactor = 0.5
    with pytest.raises(B200PTError):
        PathTracer(0).onAttach(Resources(scene=scn, hdr_rgb=std_env, camera=scn.camera, size=(16, 16)))


def test_thin_walled_scattering_material_is_not_truncated(std_env, oracle_mod):
    """ADVICE r1: transmission + multiscatterColor with thicknessFactor == 0 scatters inside the medium (the device gates the
    volume walk on the scatter coefficient, like the reference) and takes more wavefront iterations than maxDepth; the host
    must keep iterating instead of dropping the paths still queued.  Image mean and ray budgets against the oracle (the
    random walk itself is chaotic, see test_render_parity_glass_volume_scatter_statistical)."""
    from vk_gltf_renderer_b200 import synth
    scn = synth.synth_glass(n=32, scatter=True)
    scn.materials[0].thicknessFactor = 0.0
    o = _oracle(oracle_mod, scn, std_env)
    ref = oracle_mod.render(o, scn.camera, 96, 96, 8, max_depth=4)
    pt, img = _gpu_render(scn, std_env, 96, 96, 8, ptMaxDepth=4)
    assert np.isfinite(img).all()
    st, so = pt.stats(), o.stats()
    assert abs(st["closestRays"] / so["closestRays"] - 1.0) <= 1e-2
    assert abs(img[..., :3].mean() / ref[..., :3].mean() - 1.0) <= 2e-2


def test_malformed_scene_is_rejected(box_scene, std_env):
    """Out-of-range indices / material ids / texture slots return B200PT_E_INVALID instead of reading out of bounds; so do
    textures the device cannot sample like the reference: a side of 65536 or more (a 17th mip level, beyond the 16 the
    device stores) and sampler enums getSampler does not map."""
    import copy
    from vk_gltf_renderer_b200 import synth
    from vk_gltf_renderer_b200.renderer import B200PTError, PathTracer, Resources
    tex = {"tex_65536x1": (np.zeros((1, 65536, 4), np.uint8), {}), "tex_1x65536": (np.zeros((65536, 1, 4), np.uint8), {}),
           "wrap": (np.zeros((4, 4, 4), np.uint8), dict(wrapT=33069)), "mag": (np.zeros((4, 4, 4), np.uint8), dict(magFilter=9730)),
           "min": (np.zeros((4, 4, 4), np.uint8), dict(minFilter=9983))}
    for what in ("index", "material", "slot") + tuple(tex):
        scn = synth.scene_from_state(copy.deepcopy(synth.scene_state(box_scene)))
        if what == "index":
            scn.render_prims[0]["indices"] = scn.render_prims[0]["indices"].copy()
            scn.render_prims[0]["indices"][0, 0] = 1 << 20
        elif what == "material":
            scn.render_nodes[0]["materialID"] = 99
        elif what == "slot":
            scn.materials[0].pbrBaseColorTexture = 77
        else:
            scn.add_texture(tex[what][0], **tex[what][1])
        pt = PathTracer(0)
        with pytest.raises(B200PTError, match="65536" if what.startswith("tex") else None):
            pt.onAttach(Resources(scene=scn, hdr_rgb=std_env, camera=scn.camera, size=(16, 16)))
    # the largest texture the device does store: a side of 32768, 16 levels, the coarsest one sampled beyond the chain
    scn = synth.scene_from_state(copy.deepcopy(synth.scene_state(box_scene)))
    img = np.zeros((1, 32768, 4), np.uint8)
    img[..., 3] = 255
    scn.add_texture(img, magFilter=9728)
    PathTracer(0).onAttach(Resources(scene=scn, hdr_rgb=std_env, camera=scn.camera, size=(16, 16)))


def test_selection_ids_and_ndc_depth_of_frame_zero(std_env, oracle_mod):
    """traceSelectionRay / TraceLow (pixel-centre ray, every triangle opaque, no culling -> render node + 1) and the NDC depth
    of the first hit, written on the first frame of an accumulation (gltf_pathtrace.slang:604-616,
    raytracer_interface.h.slang:124-137): ids exact, depth to rounding, on a scene with MASK foliage in front of walls
    (the selection ray stops at a leaf quad the alpha test lets the camera ray pass) and one with several samples per pixel."""
    from vk_gltf_renderer_b200 import camera as cm, synth
    from vk_gltf_renderer_b200.renderer import PathTracer, Resources
    for scn, spp in ((synth.synth_sponza(tex_size=64, detail=0.05), 1), (synth.synth_material_zoo(), 3)):
        w, h = 160, 96
        o = _oracle(oracle_mod, scn, std_env)
        fi = cm.make_frame_info(scn.camera, w, h)
        pc = cm.make_push_constant(scn.camera, h, frame_count=0, total_samples=0, num_samples=spp, max_depth=4)
        acc = np.zeros((h, w, 4), np.float32)
        ids_ref, depth_ref = np.zeros((h, w), np.uint32), np.zeros((h, w), np.float32)
        o.render_frame(fi, pc, acc, object_id=ids_ref, ndc_depth=depth_ref)
        res = Resources(scene=scn, hdr_rgb=std_env, camera=scn.camera, size=(w, h))
        pt = PathTracer(0)
        pt.ptMaxDepth, pt.ptSamples = 4, spp
        pt.onAttach(res)
        for f in range(3):  # later frames must leave the frame-0 images alone
            res.frameCount = f
            pt.onRender(None, res)
        ids, depth = pt.read_selection()
        assert np.array_equal(ids, ids_ref)
        assert np.allclose(depth, depth_ref, rtol=0, atol=2e-6)
        assert 0 < (ids == 0).mean() < 0.9 and len(np.unique(ids)) > 3
        assert ((depth > 0) & (depth <= 1)).all() and (depth[ids_ref == 0] == 1.0).mean() > 0.5
        pt.onDetach(res)


def test_render_parity_infinite_plane(std_env, oracle_mod):
    """--useInfinitePlane: the ground plane y = infinitePlaneDistance with its own base colour / metallic / roughness catches the
    rays that pass the geometry (checkInfinitePlaneIntersection, pathtrace_functions.h.slang:556-585; material swap
    gltf_pathtrace.slang:165-173): stream-replicated parity with the oracle, the plane is visible."""
    from vk_gltf_renderer_b200 import synth
    from vk_gltf_renderer_b200.renderer import B200PTError, PathTracer, Resources
    scn = synth.synth_material_zoo()
    scn.render_nodes = scn.render_nodes[:-1]  # drop the zoo's own floor: the infinite plane takes its place
    kw = dict(infinite_plane=True, plane_distance=-0.02, plane_color=(0.7, 0.5, 0.3), plane_metallic=0.1, plane_roughness=0.4)
    o = _oracle(oracle_mod, scn, std_env)
    ref = oracle_mod.render(o, scn.camera, 192, 128, 8, max_depth=6, **kw)
    res = Resources(scene=scn, hdr_rgb=std_env, camera=scn.camera, size=(192, 128))
    res.settings.useInfinitePlane, res.settings.infinitePlaneDistance, res.settings.isShadowCatcher = True, -0.02, False
    res.settings.infinitePlaneBaseColor, res.settings.infinitePlaneMetallic, res.settings.infinitePlaneRoughness = (0.7, 0.5, 0.3), 0.1, 0.4
    from vk_gltf_renderer_b200.renderer import render_headless
    pt, img = render_headless(res, 8, ptMaxDepth=6)
    e = rel_rmse(img, ref)
    print("infinite plane rel RMSE", e)
    assert e <= 1e-3
    assert np.array_equal(img[..., 3] > 0, ref[..., 3] > 0)
    st, so = pt.stats(), o.stats()
    assert st["closestRays"] == so["closestRays"] and st["shadedHits"] == so["shadedHits"]
    res2 = Resources(scene=scn, hdr_rgb=std_env, camera=scn.camera, size=(192, 128))
    _, bare = render_headless(res2, 2, ptMaxDepth=6)
    assert (img[100:, :, 3] > 0).mean() > 0.9 and (bare[100:, :, 3] > 0).mean() < 0.6   # the lower image rows now hit the plane


def test_render_parity_shadow_catcher(std_env, oracle_mod):
    """The reference's default plane mode (isShadowCatcher, src/resources.hpp:112): the plane shows the environment behind it, darkened
    where a light sample is blocked, and shadowed hits continue with bsdfSampleSimple without consuming depth (handleShadowCatcher,
    pathtrace_functions.h.slang:499-554; eEarlyContinue, gltf_pathtrace.slang:176-185).  Punctual lights + environment, a MASK
    foliage scene (coloured / stochastic shadow transmission through the any-hit kernels), 2 samples per pixel, frame batching, a
    non-zero shadowCatcherDarkness: stream-replicated parity with the oracle, identical ray budgets, and the catcher is visibly not
    the solid plane."""
    from vk_gltf_renderer_b200 import synth
    from vk_gltf_renderer_b200.renderer import PathTracer, Resources, render_headless
    lit = synth.synth_lit()
    lit.render_nodes = lit.render_nodes[1:]          # drop the floor: the catcher plane replaces it
    zoo = synth.synth_material_zoo()
    zoo.render_nodes = zoo.render_nodes[:-1]
    for name, scn, dist, dark in (("lit", lit, -0.01, 0.0), ("zoo", zoo, -0.02, 0.35)):
        kw = dict(infinite_plane=True, plane_distance=dist, plane_color=(0.6, 0.6, 0.55), plane_metallic=0.2, plane_roughness=0.35, shadow_catcher=True,
                  catcher_darkness=dark)
        o = _oracle(oracle_mod, scn, std_env)
        ref = oracle_mod.render(o, scn.camera, 192, 128, 6, max_depth=5, num_samples=2, **kw)
        res = Resources(scene=scn, hdr_rgb=std_env, camera=scn.camera, size=(192, 128))
        res.settings.useInfinitePlane, res.settings.infinitePlaneDistance, res.settings.shadowCatcherDarkness = True, dist, dark
        res.settings.infinitePlaneBaseColor, res.settings.infinitePlaneMetallic, res.settings.infinitePlaneRoughness = (0.6, 0.6, 0.55), 0.2, 0.35
        assert res.settings.isShadowCatcher                      # the reference's default
        pt = PathTracer(0)
        pt.ptMaxDepth, pt.ptSamples = 5, 2
        pt.onAttach(res)
        pt.set_frame_batch(3)
        for f in range(6):
            res.frameCount = f
            pt.onRender(None, res)
        img = pt.read_accum()
        e = rel_rmse(img, ref)
        print("shadow catcher", name, "rel RMSE", e)
        assert np.isfinite(img).all() and e <= 1e-3
        st, so = pt.stats(), o.stats()
        assert st["closestRays"] == so["closestRays"] and st["shadowRays"] == so["shadowRays"] and st["shadedHits"] == so["shadedHits"]
        # against the solid plane: different picture (the catcher is see-through where lit)
        res.settings.isShadowCatcher = False
        _, solid = render_headless(res, 2, ptMaxDepth=5)
        ok = np.isfinite(solid).all(-1)   # (a sphere light seen from > 1 km gives the restated nvshaders light sample an infinite pdf in both
        assert ok.mean() > 0.99          #  implementations: a handful of NaN pixels at the horizon of the SOLID plane, none with the catcher)
        assert rel_rmse(img[ok], solid[ok]) > 0.05
        pt.onDetach(res)


def test_refit_after_transform_update_matches_a_fresh_build(std_env, oracle_mod):
    """b200pt_update_transforms (the TLAS-update / refit analogue, src/gltf_scene_rtx.cpp:416-503): three render nodes of the lit
    scene are moved, rotated, one mirrored; the device recomputes the triangle records and refits the three trees bottom-up.
    Ray-level hits (closest + shadow, with any-hit seeds on the alpha scene) and the rendered image must equal the oracle's on the
    moved scene -- i.e. exactly what a fresh build gives."""
    import copy
    import torch
    from gpu_util import random_rays, to_dev
    from vk_gltf_renderer_b200 import scene as scene_mod, synth
    from vk_gltf_renderer_b200.renderer import PathTracer, Resources

    def move(scn, k, m):
        rn = scn.render_nodes[k]
        cur = np.asarray(rn["objectToWorld"], np.float64).reshape(4, 4).T
        new = m @ cur
        rn["objectToWorld"] = scene_mod._glm(new)
        rn["worldToObject"] = scene_mod._glm(np.linalg.inv(new))
    for base, lo, hi in ((synth.synth_lit(), [-3, 0, -3], [3, 3, 3]), (synth.synth_sponza(tex_size=64, detail=0.05), [-15, 0, -6], [15, 12, 6])):
        scn = synth.scene_from_state(copy.deepcopy(synth.scene_state(base)))
        res = Resources(scene=scn, hdr_rgb=std_env, camera=scn.camera, size=(128, 96))
        pt = PathTracer(0)
        pt.ptMaxDepth = 5
        pt.onAttach(res)
        c, s_ = np.cos(0.7), np.sin(0.7)
        rot = np.array([[c, 0, s_, 0.4], [0, 1, 0, 0.3], [-s_, 0, c, -0.2], [0, 0, 0, 1.0]])
        mirror = np.diag([-1.0, 1.0, 1.0, 1.0])
        mirror[0, 3] = 0.5
        n = len(scn.render_nodes)
        move(scn, 1 % n, rot)
        move(scn, 2 % n, mirror)
        move(scn, n - 1, np.array([[1.2, 0, 0, -0.3], [0, 0.9, 0, 0.1], [0, 0, 1.1, 0.2], [0, 0, 0, 1.0]]))
        pt.update_transforms(res)
        o = _oracle(oracle_mod, scn, std_env)   # the oracle builds the moved scene from scratch
        rays = random_rays(40000, lo, hi, seed=5)
        seeds = ((np.arange(len(rays), dtype=np.uint64) * 2654435761) % (2 ** 32)).astype(np.uint32)
        s_ref = seeds.copy()
        ref = o.trace_closest(rays, s_ref)
        d_rays, d_seeds = to_dev(rays), to_dev(seeds.copy())
        d_hits = torch.empty((len(rays), 6), dtype=torch.float32, device="cuda")
        pt.trace_closest(d_rays.data_ptr(), len(rays), d_hits.data_ptr(), d_seeds.data_ptr())
        pt.synchronize()
        got = d_hits.cpu().numpy()
        assert np.array_equal(got.view(np.uint32)[:, 1:4], ref.view(np.uint32)[:, 1:4])
        assert np.array_equal(got[:, [0, 4, 5]], ref[:, [0, 4, 5]]) and np.array_equal(d_seeds.cpu().numpy(), s_ref)
        rays[:, 7] = 3.0
        s_ref = seeds.copy()
        ref_t = o.trace_shadow(rays, s_ref)
        d_rays, d_seeds = to_dev(rays), to_dev(seeds.copy())
        d_t = torch.empty((len(rays), 3), dtype=torch.float32, device="cuda")
        pt.trace_shadow(d_rays.data_ptr(), len(rays), d_t.data_ptr(), d_seeds.data_ptr())
        pt.synchronize()
        assert np.array_equal(d_t.cpu().numpy(), ref_t)
        img_ref = oracle_mod.render(o, scn.camera, 128, 96, 4, max_depth=5)
        for f in range(4):
            res.frameCount = f
            pt.onRender(None, res)
        e = rel_rmse(pt.read_accum(), img_ref)
        print("refit rel RMSE", e)
        assert e <= 1e-3
        pt.onDetach(res)


def test_gpu_built_bvh_returns_the_same_hits(std_env, oracle_mod):
    """b200pt_set_bvh_builder(1): the three trees are built on the device (LBVH: Morton sort, radix tree, bottom-up fit, level-wise
    collapse to compressed 8-wide nodes).  Hits are defined in (t, triangle id) order, independent of the tree: ray-level results
    with any-hit seeds are bit-identical to the oracle (i.e. to the host-built tree) on the triangle soup and on the alpha-masked
    atrium, the rendered image agrees to 1e-3, and a refit of the device-built tree after a transform update still does."""
    import copy
    import torch
    from gpu_util import random_rays, to_dev
    from vk_gltf_renderer_b200 import scene as scene_mod, synth
    from vk_gltf_renderer_b200.renderer import PathTracer, Resources
    for base, lo, hi in ((synth.triangle_soup(20000), [-1, -1, -1], [1, 1, 1]), (synth.synth_sponza(tex_size=64, detail=0.05), [-15, 0, -6], [15, 12, 6])):
        scn = synth.scene_from_state(copy.deepcopy(synth.scene_state(base)))
        if scn.camera is None:
            scn.camera = synth.synth_lit().camera
        res = Resources(scene=scn, hdr_rgb=std_env, camera=scn.camera, size=(128, 96))
        pt = PathTracer(0)
        pt.ptMaxDepth = 5
        pt.onAttach(res)
        host_ms = pt.bvh_build_ms()
        pt.set_bvh_builder(1)
        pt.onSceneInvalidated(res)
        print("BVH build: host %.1f ms, device %.1f ms (%d triangles)" % (host_ms, pt.bvh_build_ms(), scn.num_triangles()))
        for moved in (False, True):
            if moved:
                rn = scn.render_nodes[len(scn.render_nodes) - 1]
                m = np.asarray(rn["objectToWorld"], np.float64).reshape(4, 4).T
                m = np.array([[0.9, 0, 0.2, 0.15], [0, 1.1, 0, 0.05], [-0.2, 0, 0.9, -0.1], [0, 0, 0, 1.0]]) @ m
                rn["objectToWorld"], rn["worldToObject"] = scene_mod._glm(m), scene_mod._glm(np.linalg.inv(m))
                pt.update_transforms(res)
            o = _oracle(oracle_mod, scn, std_env)
            rays = random_rays(40000, lo, hi, seed=9)
            seeds = ((np.arange(len(rays), dtype=np.uint64) * 2654435761) % (2 ** 32)).astype(np.uint32)
            s_ref = seeds.copy()
            ref = o.trace_closest(rays, s_ref)
            d_rays, d_seeds = to_dev(rays), to_dev(seeds.copy())
            d_hits = torch.empty((len(rays), 6), dtype=torch.float32, device="cuda")
            pt.trace_closest(d_rays.data_ptr(), len(rays), d_hits.data_ptr(), d_seeds.data_ptr())
            pt.synchronize()
            got = d_hits.cpu().numpy()
            assert np.array_equal(got.view(np.uint32)[:, 1:4], ref.view(np.uint32)[:, 1:4])
            assert np.array_equal(got[:, [0, 4, 5]], ref[:, [0, 4, 5]]) and np.array_equal(d_seeds.cpu().numpy(), s_ref)
            rays[:, 7] = 3.0
            s_ref = seeds.copy()
            ref_t = o.trace_shadow(rays, s_ref)
            d_rays, d_seeds = to_dev(rays), to_dev(seeds.copy())
            d_t = torch.empty((len(rays), 3), dtype=torch.float32, device="cuda")
            pt.trace_shadow(d_rays.data_ptr(), len(rays), d_t.data_ptr(), d_seeds.data_ptr())
            pt.synchronize()
            assert np.array_equal(d_t.cpu().numpy(), ref_t)
        img_ref = oracle_mod.render(o, scn.camera, 128, 96, 3, max_depth=5)
        for f in range(3):
            res.frameCount = f
            pt.onRender(None, res)
        assert rel_rmse(pt.read_accum(), img_ref) <= 1e-3
        pt.onDetach(res)
