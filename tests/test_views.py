"""CPU: the views entry points (b200pt_set_views, b200pt_render_views, b200pt_read_views, b200pt_get_views_device) are declared,
bound and exported, and camera.view_frame_infos builds frame infos that differ from their base only in the pose fields."""
import ctypes as C
import math
import os
import re

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VIEW_ENTRY_POINTS = ("b200pt_set_views", "b200pt_render_views", "b200pt_read_views", "b200pt_get_views_device")


def test_view_entry_points_are_declared_bound_and_exported():
    from vk_gltf_renderer_b200 import _lib, abi
    hdr = open(os.path.join(ROOT, "include", "b200pt.h")).read()
    L = _lib.lib()
    for name in VIEW_ENTRY_POINTS:
        assert re.search(r"\bint " + name + r"\(", hdr), name
        assert name in _lib.EXPORTS and getattr(L, name).argtypes, name
    assert L.b200pt_render_views.argtypes[1] is C.POINTER(abi.FrameInfo)
    assert abi.MAX_VIEWS == 64
    assert set(abi.VIEW_POSE_FIELDS) <= {n for n, _ in abi.FrameInfo._fields_}


def _non_pose_bytes(fi):
    from vk_gltf_renderer_b200 import abi
    raw = bytearray(bytes(fi))
    for name in abi.VIEW_POSE_FIELDS:
        f = getattr(abi.FrameInfo, name)
        raw[f.offset:f.offset + f.size] = b"\0" * f.size
    return bytes(raw)


def test_view_frame_infos_change_only_the_pose():
    from vk_gltf_renderer_b200 import abi, camera
    from vk_gltf_renderer_b200.scene import Camera
    cam = Camera()
    cam.eye, cam.center = np.array([0.3, 1.2, 4.0], np.float32), np.array([0.0, 0.5, 0.0], np.float32)
    base = camera.make_frame_info(cam, 320, 200, infinite_plane=True, plane_distance=-0.25, shadow_catcher=True, catcher_darkness=0.3,
                                  env_rotation=0.7, env_intensity=1.5)
    base.jitter[:] = [0.125, -0.25]
    views = [camera.look_at((4.0 * math.sin(a), 1.2, 4.0 * math.cos(a)), cam.center, cam.up) for a in np.linspace(0.0, 2.0, 6)]
    fis = camera.view_frame_infos(base, views)
    assert len(fis) == 6
    proj = camera.perspective_vk(cam.yfov, 320 / 200.0, cam.znear, cam.zfar)
    for fi, view in zip(fis, views):
        assert _non_pose_bytes(fi) == _non_pose_bytes(base)
        glm = lambda name: np.asarray(getattr(fi, name), np.float64).reshape(4, 4).T  # noqa: E731
        assert np.allclose(glm("viewMatrix"), view, atol=1e-6)
        assert np.allclose(glm("viewInv") @ view, np.eye(4), atol=1e-5)
        assert np.allclose(glm("viewProjMatrix"), proj @ view, rtol=1e-5, atol=1e-5)
        assert bytes(fi.prevMVP) == bytes(fi.viewProjMatrix)
    assert bytes(fis[0].viewMatrix) != bytes(fis[1].viewMatrix)
    # the views' pose is all that differs between them
    assert len({_non_pose_bytes(fi) for fi in fis}) == 1
    # the base is not modified
    assert bytes(base.viewMatrix) == bytes(camera.make_frame_info(cam, 320, 200).viewMatrix)
    assert isinstance(fis, C.Array) and fis._type_ is abi.FrameInfo
