"""Camera math + per-frame structs for the path tracer boundary.

Mirrors what GltfRenderer::onRender writes into SceneFrameInfo every frame
(reference src/renderer.cpp:675-705) and PathTracer::setupPushConstant into the push constants
(src/renderer_pathtracer.cpp:1496-1574).  nvutils::CameraManipulator is external (nvpro_core2);
its matrices are glm::lookAt and glm::perspectiveRH_ZO with the Vulkan Y flip ([1][1] *= -1).
All arithmetic is done in float64 and rounded once to float32.
"""
import ctypes as C
import math

import numpy as np

from . import abi


def look_at(eye, center, up):
    eye, center, up = (np.asarray(v, np.float64) for v in (eye, center, up))
    f = center - eye
    f /= np.linalg.norm(f)
    s = np.cross(f, up)
    s /= np.linalg.norm(s)
    u = np.cross(s, f)
    m = np.eye(4)
    m[0, :3], m[1, :3], m[2, :3] = s, u, -f
    m[0, 3], m[1, 3], m[2, 3] = -s @ eye, -u @ eye, f @ eye
    return m


def perspective_vk(yfov, aspect, znear, zfar):
    t = math.tan(yfov / 2.0)
    m = np.zeros((4, 4))
    m[0, 0] = 1.0 / (aspect * t)
    m[1, 1] = -1.0 / t  # Vulkan clip space: +Y down
    m[2, 2] = zfar / (znear - zfar)
    m[3, 2] = -1.0
    m[2, 3] = -(zfar * znear) / (zfar - znear)
    return m


def ortho_vk(xmag, ymag, znear, zfar):
    m = np.eye(4)
    m[0, 0] = 1.0 / xmag
    m[1, 1] = -1.0 / ymag
    m[2, 2] = -1.0 / (zfar - znear)
    m[2, 3] = -znear / (zfar - znear)
    return m


def fit_camera(lo, hi, yfov=math.radians(45.0), aspect=1.0):
    """CameraManipulator::fit(bbox) analogue used when the glTF has no camera
    (gltf_camera_utils.hpp:80-86): look at the box centre from +Z far enough to see the bounding sphere."""
    from .scene import Camera
    lo, hi = np.asarray(lo, np.float64), np.asarray(hi, np.float64)
    c = (lo + hi) * 0.5
    r = float(np.linalg.norm(hi - lo) * 0.5)
    cam = Camera()
    cam.yfov = yfov
    d = r / math.sin(min(yfov, 2 * math.atan(math.tan(yfov / 2) * aspect)) / 2.0)
    cam.eye = (c + np.array([0, 0, d])).astype(np.float32)
    cam.center = c.astype(np.float32)
    cam.znear, cam.zfar = 0.001 * r, 100.0 * r
    return cam


def _glm(m):
    return np.ascontiguousarray(np.asarray(m, np.float64).T.reshape(16), np.float32)


def make_frame_info(cam, width, height, *, use_hdr=True, env_rotation=0.0, env_intensity=1.0, env_blur=0.0,
                    solid_background=False, background=(0, 0, 0), infinite_plane=False, plane_distance=0.0,
                    plane_color=(0.5, 0.5, 0.5), plane_metallic=0.0, plane_roughness=0.5, shadow_catcher=False, catcher_darkness=0.0):
    """SceneFrameInfo as filled at src/renderer.cpp:677-700 (projection uses the *window* aspect)."""
    view = look_at(cam.eye, cam.center, cam.up)
    if cam.type == "orthographic":
        proj = ortho_vk(cam.xmag, cam.ymag, cam.znear, cam.zfar)
    else:
        proj = perspective_vk(cam.yfov, width / float(height), cam.znear, cam.zfar)
    fi = abi.FrameInfo()
    fi.viewMatrix[:] = _glm(view).tolist()
    fi.projInv[:] = _glm(np.linalg.inv(proj)).tolist()
    fi.viewInv[:] = _glm(np.linalg.inv(view)).tolist()
    fi.viewProjMatrix[:] = _glm(proj @ view).tolist()
    fi.prevMVP[:] = _glm(proj @ view).tolist()
    fi.jitter[:] = [0.0, 0.0]
    fi.imageSize[:] = [float(width), float(height)]
    fi.flags = ((abi.SCENE_IS_ORTHOGRAPHIC if cam.type == "orthographic" else 0)
                | (abi.SCENE_USE_SOLID_BACKGROUND if solid_background else 0)
                | (abi.SCENE_USE_HDR_ENVIRONMENT if use_hdr else 0)
                | (abi.SCENE_USE_INFINITE_PLANE if infinite_plane else 0)
                | (abi.SCENE_INFINITE_PLANE_SHADOW_CATCHER if (infinite_plane and shadow_catcher) else 0))
    fi.envRotation = env_rotation
    fi.envBlur = env_blur
    fi.envIntensity = env_intensity
    fi.backgroundColor[:] = list(background)
    fi.visualization = 0
    fi.infinitePlaneDistance = plane_distance
    fi.infinitePlaneBaseColor[:] = list(plane_color)
    fi.infinitePlaneMetallic = plane_metallic
    fi.infinitePlaneRoughness = plane_roughness
    fi.shadowCatcherDarkenAmount = max(catcher_darkness, 0.0)   # src/renderer.cpp:700
    return fi


def view_frame_infos(base, views):
    """The frame infos of b200pt_render_views: one copy of `base` per view, with that view's pose.  `views` are world-to-camera
    matrices (4x4, as look_at returns them); the projection is base's (inverted from its projInv in float64), so every field but
    abi.VIEW_POSE_FIELDS is base's byte for byte.  prevMVP is the view's own viewProjMatrix (a static view)."""
    proj = np.linalg.inv(np.asarray(base.projInv, np.float64).reshape(4, 4).T)
    out = (abi.FrameInfo * len(views))()
    for fi, view in zip(out, views):
        C.memmove(C.addressof(fi), C.addressof(base), C.sizeof(abi.FrameInfo))
        view = np.asarray(view, np.float64)
        fi.viewMatrix[:] = _glm(view).tolist()
        fi.viewInv[:] = _glm(np.linalg.inv(view)).tolist()
        fi.viewProjMatrix[:] = _glm(proj @ view).tolist()
        fi.prevMVP[:] = _glm(proj @ view).tolist()
    return out


def halton(index):
    """shaderio::halton (shaders/dlss_util.h), float32 as the host evaluates it: both bases advance in one loop that stops when
    EITHER remainder reaches 0, so the base-2 digits beyond the base-3 length are not added."""
    f = np.float32
    sx = sy = f(index)
    ax, ay, az, aw = f(1.0), f(1.0), f(0.0), f(0.0)
    while sx > 0.0 and sy > 0.0:
        ax = f(ax / f(2.0))
        ay = f(ay / f(3.0))
        az = f(az + f(ax * np.fmod(sx, f(2.0))))
        aw = f(aw + f(ay * np.fmod(sy, f(3.0))))
        sx = np.floor(f(sx / f(2.0)))
        sy = np.floor(f(sy / f(3.0)))
    return az, aw


def dlss_jitter(frame_index):
    """shaderio::dlssJitter: the Halton point of the DLSS frame index, centred on (0, 0) (Dlss::beginFrame, src/dlss.cpp:401-414)"""
    hx, hy = halton(int(frame_index))
    return np.float32(hx - np.float32(0.5)), np.float32(hy - np.float32(0.5))


def make_push_constant(cam, height, *, frame_count, total_samples, num_samples=1, max_depth=5,
                       firefly_clamp=10.0, tex_grad_scale=1.0, aperture=0.0, focal_distance=None):
    """PathtracePushConstant as filled by setupPushConstant (renderer_pathtracer.cpp:1496-1574):
    autofocus focal distance = |eye - center| (:1508-1512); pixelAngle = 2|projInv[1][1]|/H (:1570-1571);
    ePtFirstFrame iff frameCount == 0 (:1542)."""
    pc = abi.PushConstant()
    pc.maxDepth = max_depth
    pc.frameCount = frame_count
    pc.fireflyClampThreshold = firefly_clamp
    pc.texGradScale = tex_grad_scale
    pc.numSamples = num_samples
    pc.totalSamples = total_samples
    pc.focalDistance = (float(np.linalg.norm(np.asarray(cam.eye, np.float64) - np.asarray(cam.center, np.float64)))
                        if focal_distance is None else focal_distance)
    pc.aperture = aperture
    pc.flags = abi.PT_FIRST_FRAME if frame_count == 0 else 0
    if cam.type == "orthographic":
        proj_inv_11 = cam.ymag
    else:
        proj_inv_11 = math.tan(cam.yfov / 2.0)
    pc.pixelAngle = np.float32(2.0 * abs(proj_inv_11) / max(float(height), 1.0))
    pc.mouseCoord[:] = [-1.0, -1.0]
    return pc
