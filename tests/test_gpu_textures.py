"""-m gpu: the device texture sampler (getTexture / sampleLevel0 in shade.cuh, through b200pt_texture_lookup) against the
oracle and the float64 Vulkan-sampler reference over the sweep of test_texture_sampling.py, the device mip chain level by
level, and the two alpha-test paths and the shade path through the production kernels on scenes whose textures use every
wrap mode, NEAREST and LINEAR filters and non-power-of-two shapes."""
import numpy as np
import pytest

import texref as tr
from conftest import rel_rmse
from gpu_util import trace_both
from test_texture_sampling import EPS, Sweep, check_chain, compare, read_levels, reference
from vk_gltf_renderer_b200 import tex_io

pytestmark = pytest.mark.gpu


def _device(scene):
    from vk_gltf_renderer_b200.renderer import PathTracer, Resources
    from vk_gltf_renderer_b200.scene import Camera
    pt = PathTracer(0)
    pt.onAttach(Resources(scene=scene, camera=scene.camera or Camera(), size=(8, 8)))
    return pt


def _lookup(pt):
    import torch

    def f(records):
        records = np.ascontiguousarray(records, np.float32).reshape(-1, 8)
        d_in = torch.from_numpy(records).cuda()
        d_out = torch.empty((len(records), 4), dtype=torch.float32, device="cuda")
        pt.texture_lookup(d_in.data_ptr(), len(records), d_out.data_ptr())
        pt.synchronize()
        return d_out.cpu().numpy()
    return f


def test_device_sampler_matches_oracle_and_float64_reference(oracle_mod):
    from vk_gltf_renderer_b200.renderer import B200PTError
    sweep = Sweep()
    pt = _device(sweep.scene)
    dev = _lookup(pt)
    o = oracle_mod.Oracle()
    o.set_scene(sweep.scene)
    # the device chain, level by level (packTiled's 4x4 tiles, padded narrow levels, levelOfs): the float64 blit of the
    # stored previous level, and the very same bytes as the oracle's chain
    stored, ties = {}, 0
    for k, im in enumerate(sweep.images):
        levels, beyond = read_levels(dev, sweep, im)
        ties += check_chain(levels, beyond, im)
        ref_levels, _ = read_levels(o.texture_lookup, sweep, im)
        assert all(np.array_equal(a, b) for a, b in zip(levels, ref_levels)), (im["w"], im["h"], im["srgb"])
        stored[k] = levels
    print("device mip chain: texels one step off the float64 blit on a tie:", ties)

    got, want = dev(sweep.queries), o.texture_lookup(sweep.queries)
    ref, alt, lam, edge = reference(sweep, stored)
    print("device vs texref:", compare(got, ref, alt, lam, edge, "device"))
    # bit for bit wherever the result does not go through log2f: level 0 (mode 1, no gradient) and magnification
    no_log = ~(lam > -EPS)
    assert no_log.sum() > 0.5 * len(got)
    assert np.array_equal(got[no_log].view(np.uint32), want[no_log].view(np.uint32))
    # with a gradient: CUDA's log2f and libm's may differ by an ulp.  Off a boundary that moves only the weight of a linear
    # mip blend (a difference ~1e-7 of the two levels' gap) -- a nearest level selection is unaffected and stays bit for
    # bit; on a boundary it may select the other side (checked against texref above).
    grad = (lam > -EPS) & ~edge
    blend = np.concatenate([np.full(m["n"], m["kind"] == "grad" and tr.sampler_modes(*sweep.textures[m["tex"]]["state"][2:])[2])
                            for m in sweep.meta]) & grad
    diff = np.abs(got - want).max(1)
    moved = grad & (diff > 0)
    flips = edge & (diff > 0)
    print("gradient queries: %d (%d of them linear mip blends); differing by a log2f ulp off a boundary: %d; on a lambda "
          "boundary: %d, of which differ: %d" % (grad.sum(), blend.sum(), moved.sum(), edge.sum(), flips.sum()))
    assert not (moved & ~blend).any(), np.flatnonzero(moved & ~blend)[:5]
    assert (diff[grad] <= 1e-6).all(), diff[grad].max()
    # a slot outside the scene's texture infos and a mode other than 0 / 1 are refused before any launch
    for bad in (tex_io.records(len(sweep.scene.texture_infos), [[0.5, 0.5]]), tex_io.records(1, [[0.5, 0.5]], mode=2)):
        with pytest.raises(B200PTError):
            dev(bad)
    pt.onDetach()


def test_alpha_paths_with_every_sampler_state(oracle_mod):
    """14 stacked alpha layers, each with its own texture shape and sampler (synth.sampler_layers): the pre-gathered
    alpha records (opacityFromRecord) and, past the candidate budget, the generic getOpacity fallback decide every
    candidate like the oracle -- ids, t, u, v, seeds and shadow transmission bit for bit."""
    from gpu_util import random_rays
    from vk_gltf_renderer_b200 import synth
    scn = synth.sampler_layers()
    pt = _device(scn)
    o = oracle_mod.Oracle()
    o.set_scene(scn)
    rays = random_rays(60000, [-1.6, 0.1, -2.2], [1.9, 2.1, 0.2])
    seeds = ((np.arange(len(rays), dtype=np.uint64) * 2654435761) % (2 ** 32)).astype(np.uint32)
    ref, _, ref_t, _ = trace_both(pt, o, rays, seeds, float_cols=(0, 4, 5))
    node = ref.view(np.int32)[:, 1]
    layer_hit = (node >= 0) & (node < 14)
    assert 0.1 < layer_hit.mean() < 0.9 and len(np.unique(node[layer_hit])) == 14
    assert 0.02 < (ref_t[:, 0] > 0).mean() < 0.98
    pt.onDetach()


def test_shade_path_with_clamped_mirrored_nearest_and_transformed_textures(std_env, oracle_mod):
    """The material zoo with a clamped x mirrored non-power-of-two base colour under a rotated, scaled texture transform and a
    NEAREST metallic-roughness texture: image parity, and the first-hit albedo of the guide image -- a per-pixel readout of
    getTexture -- like test_gpu_guides."""
    from test_guides import render_with_guide
    from vk_gltf_renderer_b200 import synth
    from vk_gltf_renderer_b200.renderer import PathTracer, Resources
    scn = synth.synth_material_zoo(samplers=True)
    o = oracle_mod.Oracle()
    o.set_scene(scn)
    o.set_environment(std_env)
    W, H = 192, 128
    res = Resources(scene=scn, hdr_rgb=std_env, camera=scn.camera, size=(W, H))
    pt = PathTracer(0)
    pt.ptMaxDepth = 4
    pt.ptSamples = 2
    pt.onAttach(res)
    pt.ptUseOptixDenoiser = True
    pt.set_guide_outputs(True)
    for f in range(3):
        res.frameCount = f
        pt.onRender(None, res)
    img = pt.read_accum()
    albedo, _ = pt.read_guide()
    ref_img, ref_albedo, _ = render_with_guide(oracle_mod, o, scn.camera, W, H, 3, num_samples=2, max_depth=4)
    e = rel_rmse(img, ref_img)
    same = (albedo == ref_albedo).all(-1)
    print("sampler zoo rel RMSE", e, "albedo equal", same.mean())
    assert e <= 1e-3
    assert same.mean() > 0.995 and np.abs(albedo - ref_albedo).max() < 2e-3
    assert (ref_albedo != 0).any(-1).mean() > 0.4
    pt.onDetach(res)
