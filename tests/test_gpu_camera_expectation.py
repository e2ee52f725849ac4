"""The device's camera stage against the float64 model of tests/camref.py: the cases of test_camera_expectation.py at 256 x 192
through render_headless, a frame batch of 3 with frames in flight, a row tile and an interleaved band, three camera poses through
render_views, and DLSS frames at a fixed jitter."""
import numpy as np
import pytest

import camcases as CC
from vk_gltf_renderer_b200 import abi, tiling
from vk_gltf_renderer_b200 import camera as camm
from vk_gltf_renderer_b200.renderer import PathTracer, Resources, render_headless

pytestmark = pytest.mark.gpu

W, H = 256, 192
FRAMES = 256
LENS_PIXELS = 1500
ORDER_TOL = 5e-4


def _render(case, frames, tile=None, batch=1, lanes=1):
    cam = CC.camera(case["cam"])
    scn, tris = CC.build_scene(cam, W, H, case["back"])
    res = Resources(scene=scn, hdr_rgb=CC.env_image(), camera=cam, size=(W, H), tile=tile)
    res.settings.useSolidBackground = case["back"] == "solid"
    res.settings.solidBackgroundColor = CC.BACKGROUND
    pt = PathTracer(0)
    pt.ptMaxDepth, pt.ptSamples = 4, case["spp"]
    pt.ptFireflyClamp = case.get("clamp", CC.NO_CLAMP)
    pt.ptAperture = case.get("aperture", 0.0)
    pt.onAttach(res)
    pt.set_frames_in_flight(lanes)
    pt.set_frame_batch(batch)
    pt, img = render_headless(res, frames, pt=pt)
    ids, depth = pt.read_selection()
    pt.onDetach()
    return cam, tris, img, ids, depth


def _check(case, cam, tris, img, ids, depth, row_ids, label, frames=FRAMES, view_cam=None):
    model = CC.make_model(cam, W, H, case, tris, view_cam=view_cam)
    ex = CC.Expectation(model, case["spp"], frames, row_ids, max_mixed=LENS_PIXELS if model.lens else None)
    report = []
    fails = CC.check_image(ex, img, label, report, case.get("clamp", CC.NO_CLAMP))
    fails += CC.check_selection(ex, ids, label, back_id=4 if case["back"] == "tri" else 0)
    if depth is not None:
        fails += CC.check_depth(ex, depth, cam, case, label)
    report.append(f"{label}: lens quadrature orders differ by {ex.order_gap:.2e} (largest region value {np.abs(model.vals).max():.2f})")
    print("\n".join(report))
    assert ex.order_gap <= ORDER_TOL * np.abs(model.vals).max(), ex.order_gap
    assert not fails, "\n".join(fails)


@pytest.mark.parametrize("name", sorted(CC.CASES))
def test_gpu_camera(name):
    case = CC.resolve(CC.CASES[name], H)
    _check(case, *_render(case, FRAMES), np.arange(H), name)


@pytest.mark.parametrize("spp", [1, 3])
def test_gpu_camera_batch(spp):
    """a frame batch of 3 with two frames in flight: each frame of a batch keeps its own seed and sample count"""
    case = CC.resolve(CC.CASES[f"lens_rot_spp{spp}"], H)
    _check(case, *_render(case, FRAMES, batch=3, lanes=2), np.arange(H), f"batch3 spp{spp}")


@pytest.mark.parametrize("tile", [(37, 71), ("interleave", 8, 2, 1)])
def test_gpu_camera_tile(tile):
    """getRay takes the global row and the full frame's imageSize; a strip has fewer edge pixels, so it runs twice the frames"""
    case = CC.resolve(CC.CASES["lens_rot_spp1"], H)
    rows = (np.arange(tile[0], tile[0] + tile[1]) if tile[0] != "interleave"
            else np.asarray(tiling.interleaved_rows(H, tile[2], tile[3], tile[1])))
    _check(case, *_render(case, 2 * FRAMES, tile=tile), rows, f"tile {tile}", frames=2 * FRAMES)


def view_cameras():
    """three poses of the lens case: the rotated camera, the axis-aligned control and a third turned the other way, all at the
    rotated camera's distance from the look-at point so that one focal distance fits them"""
    base = CC.camera("rot")
    ctrl = CC.camera("axis")
    ctrl.center = base.center.copy()
    ctrl.eye = (np.asarray(base.center, np.float64) + [0.0, 0.0, CC.focal(base)]).astype(np.float32)
    third = CC.camera("rot")
    third.eye = (np.asarray(base.center, np.float64) + CC.focal(base) * np.array([-0.1, 0.1, 0.99]) / np.linalg.norm([-0.1, 0.1, 0.99])).astype(np.float32)
    return [base, ctrl, third]


def test_gpu_camera_views():
    """render_views: each view's rays and lens come from its own pose, and each view converges to its own expectation.  The
    views' edge bands are narrower than view 0's, so the test runs twice the frames."""
    case = CC.resolve(CC.CASES["lens_rot_spp1"], H)
    cams = view_cameras()
    scn, tris = CC.build_scene(cams[0], W, H, case["back"])
    res = Resources(scene=scn, hdr_rgb=CC.env_image(), camera=cams[0], size=(W, H))
    pt = PathTracer(0)
    pt.onAttach(res)
    pt.set_views(len(cams))
    base = CC.frame_info(cams[0], W, H, case)
    fis = camm.view_frame_infos(base, [camm.look_at(c.eye, c.center, c.up) for c in cams])
    frames = 2 * FRAMES
    for f in range(frames):
        pt.render_views(fis, CC.push_constant(cams[0], H, case, f, 1))
    rgba, ids, depth = pt.read_views()
    pt.onDetach()
    for v, c in enumerate(cams):
        # the triangles face view 0 only: the NDC depth check needs fronto-parallel triangles
        _check(case, cams[0], tris, rgba[v], ids[v], depth[v] if v == 0 else None, np.arange(H), f"view {v}", frames=frames, view_cam=c)


@pytest.mark.parametrize("name", sorted(CC.DLSS))
def test_gpu_camera_dlss(name):
    """DLSS frames (set_dlss_guides) sample at 0.5 + the frame's jitter without the Gaussian draws and replace the image.
    Without an aperture the image is deterministic; with one, the replaced images of frames at one jitter average to the
    lens-only expectation."""
    case = CC.resolve(CC.DLSS[name], H)
    cam = CC.camera(case["cam"])
    scn, tris = CC.build_scene(cam, W, H, case["back"])
    res = Resources(scene=scn, hdr_rgb=CC.env_image(), camera=cam, size=(W, H))
    pt = PathTracer(0)
    pt.onAttach(res)
    pt.set_dlss_guides(True)
    fi = CC.frame_info(cam, W, H, case)
    fi.jitter[:] = list(CC.DLSS_JITTER)
    frames = FRAMES if case.get("lens") else 1
    total = np.zeros((H, W, 4))
    for f in range(frames):
        pc = CC.push_constant(cam, H, case, f, 1)
        pc.flags |= abi.PT_USE_DLSS
        pt.render_frame_raw(fi, pc)
        img = pt.read_accum()
        total += img
    pt.onDetach()
    model = CC.make_model(cam, W, H, case, tris)
    off = CC.dlss_offset(fi)
    if not model.lens:
        fails = CC.check_dlss_point(model, img, off, np.arange(H), name)
        assert not fails, "\n".join(fails)
        return
    ex = CC.Expectation(model, 1, frames, np.arange(H), max_mixed=LENS_PIXELS, dlss_offset=off)
    report = []
    fails = CC.check_image(ex, total / frames, name, report)
    print("\n".join(report))
    assert not fails, "\n".join(fails)
