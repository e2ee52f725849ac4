"""GPU: b200pt_set_views / b200pt_render_views render several camera poses of one frame as one wavefront, each into its own
images.  Every view's image, object ids and depth must be bit-identical to rendering that view alone with b200pt_render_frame over
the same push-constant sequence, and the ray counters must be the sums of those renders."""
import ctypes as C
import math

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

W, H = 64, 48
E_INVALID, E_UNSUPPORTED = -1, -4
COUNTERS = ("closestRays", "shadowRays", "shadedHits", "pathsStarted")


@pytest.fixture(scope="module")
def scenes():
    from vk_gltf_renderer_b200 import synth
    # alpha-MASK foliage under the infinite plane, transmission through a scattering volume, punctual lights
    return {"sponza_plane": synth.synth_sponza(tex_size=128, detail=0.05), "glass_volume": synth.synth_glass(scatter=True),
            "lit": synth.synth_lit()}


def _tracer(scn, env, lanes, tile=None, size=(W, H)):
    from vk_gltf_renderer_b200.renderer import PathTracer, Resources
    res = Resources(scene=scn, hdr_rgb=env, camera=scn.camera, size=size, tile=tile)
    pt = PathTracer(0)
    pt.onAttach(res)
    pt.set_frames_in_flight(lanes)
    return pt, res


def _frame_infos(scn, n, plane, size=(W, H)):
    """n poses: the scene camera's eye turned about the look-at point, a few degrees apart"""
    from vk_gltf_renderer_b200 import camera
    cam = scn.camera
    base = camera.make_frame_info(cam, size[0], size[1], infinite_plane=plane, plane_distance=-0.05, shadow_catcher=False)
    eye, center = np.asarray(cam.eye, np.float64), np.asarray(cam.center, np.float64)
    views = []
    for k in range(n):
        a = math.radians(6.0 * k)
        d = eye - center
        rot = np.array([[math.cos(a), 0.0, math.sin(a)], [0.0, 1.0, 0.0], [-math.sin(a), 0.0, math.cos(a)]])
        views.append(camera.look_at(center + rot @ d, center, cam.up))
    return camera.view_frame_infos(base, views)


def _push_constants(scn, frames, spp, size=(W, H)):
    from vk_gltf_renderer_b200 import camera
    return [camera.make_push_constant(scn.camera, size[1], frame_count=f, total_samples=f * spp, num_samples=spp, max_depth=6)
            for f in range(frames)]


def _counters(pt):
    st = pt.stats()
    return np.array([st[k] for k in COUNTERS], np.int64)


def _check_views(pt, fis, pcs):
    """render_views over pcs, then every view alone with render_frame over the same pcs: equal bits and counter sums"""
    pt.reset_stats()
    for pc in pcs:
        pt.render_views(fis, pc)
    rgba, ids, depth = pt.read_views()
    got = _counters(pt)
    assert rgba.shape[0] == len(fis)
    want = np.zeros_like(got)
    for v, fi in enumerate(fis):
        pt.reset_stats()
        for pc in pcs:
            pt.render_frame_raw(fi, pc)
        ref = pt.read_accum()
        ref_ids, ref_depth = pt.read_selection()
        want += _counters(pt)
        assert np.array_equal(rgba[v], ref), v
        assert np.array_equal(ids[v], ref_ids) and np.array_equal(depth[v], ref_depth), v
    assert np.array_equal(got, want)
    # the poses differ, so the views do
    assert not np.array_equal(rgba[0], rgba[-1])


@pytest.mark.parametrize("scene", ["sponza_plane", "glass_volume", "lit"])
@pytest.mark.parametrize("spp,lanes,tile", [(1, 1, None), (2, 4, None), (2, 4, ("interleave", 4, 2, 1))])
def test_views_are_bit_identical_to_single_renders(scenes, std_env, scene, spp, lanes, tile):
    scn = scenes[scene]
    pt, _ = _tracer(scn, std_env, lanes, tile)
    pt.set_views(4)
    _check_views(pt, _frame_infos(scn, 4, scene == "sponza_plane"), _push_constants(scn, 3, spp))
    pt.onDetach()


def test_views_refuse_what_they_cannot_render(scenes, std_env):
    from vk_gltf_renderer_b200 import abi
    scn = scenes["lit"]
    pt, _ = _tracer(scn, std_env, 2)
    L, h = pt._L, pt._h
    pt.set_views(4)
    fis = _frame_infos(scn, 4, False)
    pc = _push_constants(scn, 1, 1)[0]
    # a field other than the pose differs
    bad = _frame_infos(scn, 4, False)
    bad[2].envIntensity = 0.5
    assert L.b200pt_render_views(h, bad, 4, C.byref(pc)) == E_INVALID
    bad = _frame_infos(scn, 4, False)
    bad[1].projInv[5] *= 1.01
    assert L.b200pt_render_views(h, bad, 4, C.byref(pc)) == E_INVALID
    # n differs from the view count
    assert L.b200pt_render_views(h, fis, 3, C.byref(pc)) == E_INVALID
    # the guide images of DLSS and the OptiX denoiser belong to one displayed frame
    for flag in (abi.PT_USE_DLSS, abi.PT_USE_OPTIX_DENOISER):
        p = _push_constants(scn, 1, 1)[0]
        p.flags |= flag
        assert L.b200pt_render_views(h, fis, 4, C.byref(p)) == E_UNSUPPORTED
    # frame batching and views exclude each other
    assert L.b200pt_set_frame_batch(h, 2) == E_UNSUPPORTED
    pt.set_views(1)
    pt.set_frame_batch(2)
    assert L.b200pt_set_views(h, 2) == E_UNSUPPORTED
    pt.set_frame_batch(1)
    assert L.b200pt_set_views(h, 0) == E_INVALID and L.b200pt_set_views(h, abi.MAX_VIEWS + 1) == E_INVALID
    # the handle still renders views correctly
    pt.set_views(4)
    _check_views(pt, fis, _push_constants(scn, 2, 1))
    pt.onDetach()


def test_views_lifecycle(scenes, std_env):
    scn = scenes["sponza_plane"]
    pcs = _push_constants(scn, 3, 1)
    fi0 = _frame_infos(scn, 1, True)[0]

    def single(pt):
        for pc in pcs:
            pt.render_frame_raw(fi0, pc)
        return (pt.read_accum(),) + pt.read_selection()

    pt, _ = _tracer(scn, std_env, 2)
    ref = single(pt)
    pt.onDetach()
    # views back to 1 render what a handle that never had views renders
    pt, res = _tracer(scn, std_env, 2)
    pt.set_views(3)
    fis = _frame_infos(scn, 3, True)
    for pc in pcs[:2]:
        pt.render_views(fis, pc)
    pt.set_views(1)
    got = single(pt)
    assert all(np.array_equal(a, b) for a, b in zip(got, ref))
    # render_frame with views set renders view 0 and leaves the other views' images alone
    pt.set_views(3)
    for pc in pcs:
        pt.render_views(fis, pc)
    before = pt.read_views()
    got = single(pt)
    assert all(np.array_equal(a, b) for a, b in zip(got, ref))
    after = pt.read_views()
    for a, b in zip(before, after):
        assert np.array_equal(a[1:], b[1:])
    # a view's device image is what read_views returns: b200pt_tonemap_image gives the same bytes for both
    import torch
    ptr, _, _ = pt.views_device_ptrs(2)
    tm = pt.make_tonemapper()
    ldr = [torch.empty((H, W, 4), dtype=torch.uint8, device="cuda") for _ in range(2)]
    host_copy = torch.from_numpy(after[0][2]).cuda()
    pt.tonemap_image(tm, ptr, W, H, ldr[0].data_ptr())
    pt.tonemap_image(tm, host_copy.data_ptr(), W, H, ldr[1].data_ptr())
    assert torch.equal(ldr[0], ldr[1]) and int(ldr[0].max()) > 0
    # a resize and a change of frames in flight keep the views
    size = (48, 32)
    pt.onResize(None, size, res)
    _check_views(pt, _frame_infos(scn, 3, True, size), _push_constants(scn, 2, 2, size))
    pt.set_frames_in_flight(3)
    _check_views(pt, _frame_infos(scn, 3, True, size), _push_constants(scn, 2, 1, size))
    pt.onDetach()
