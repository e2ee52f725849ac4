"""Host-side mirror of the reference's path-tracer backend interface.

`PathTracer` mirrors `class PathTracer : public BaseRenderer` (reference src/renderer_base.hpp:33-55,
src/renderer_pathtracer.hpp:61-88): onAttach / onDetach / onResize / onRender / onSceneInvalidated,
the `--pt*` parameters (src/renderer_pathtracer.cpp:119-132) and the public push-constant block.
`Resources` carries what the reference's `Resources` bag hands the renderer (src/resources.hpp:167-276):
scene, HDR environment, camera, settings, frame counter and the RGBA32F accumulation image.

Everything below the virtuals is one call into libb200pt.so (include/b200pt.h); there is no
CPU path here.
"""
import ctypes as C
from dataclasses import dataclass, field

import numpy as np

from . import _lib, abi, camera as cam_mod


class B200PTError(RuntimeError):
    pass


# the bytes each scene edit hands the library, by the PathTracer method that sends them: update_scene_changes sends an edit only
# when they differ from what the handle holds
_EDIT_BYTES = {
    "update_materials": lambda s: (b"".join(map(bytes, s.materials)), b"".join(map(bytes, s.texture_infos))),
    "update_lights": lambda s: b"".join(map(bytes, s.lights)),
    "set_node_visibility": lambda s: bytes(1 if rn.get("visible", True) else 0 for rn in s.render_nodes),
}


@dataclass
class Settings:
    """Resources::settings (reference src/resources.hpp:82-133) — fields the path tracer reads."""
    envSystem: int = 1            # 0 sky (not built), 1 HDR
    hdrEnvIntensity: float = 1.0
    hdrEnvRotation: float = 0.0
    hdrBlur: float = 0.0
    useSolidBackground: bool = False
    solidBackgroundColor: tuple = (0.0, 0.0, 0.0)
    maxFrames: int = 500
    useInfinitePlane: bool = False   # src/resources.hpp:111-116
    isShadowCatcher: bool = True     # the reference's default: the plane only catches shadows (src/resources.hpp:112)
    infinitePlaneDistance: float = 0.0
    infinitePlaneBaseColor: tuple = (0.5, 0.5, 0.5)
    infinitePlaneMetallic: float = 0.0
    infinitePlaneRoughness: float = 0.5
    shadowCatcherDarkness: float = 0.0   # non-physical shadow darkening (src/resources.hpp:117)


@dataclass
class Resources:
    scene: object = None          # vk_gltf_renderer_b200.scene.Scene
    hdr_rgb: np.ndarray = None    # float32 [H, W, 3]
    camera: object = None
    settings: Settings = field(default_factory=Settings)
    size: tuple = (1920, 1080)    # (width, height)
    frameCount: int = -1          # reset to -1, pre-incremented (src/renderer.cpp:1939-1977)
    tile: tuple = None            # (y0, rows) strip, or ("interleave", band_rows, world, rank); None = full image


class PathTracer:
    """Drop-in for the reference's PathTracer renderer, backed by the CUDA library."""

    def __init__(self, device=0, count_traversal=False):
        self._L = _lib.lib(count_traversal)
        self._h = C.c_void_p()
        self._device = device
        # PathtracePushConstant defaults (shaders/shaderio.h:181-190) + registerParameters names
        self.ptMaxDepth = 5
        self.ptSamples = 1
        self.ptFireflyClamp = 10.0
        self.ptTexGradScale = 1.0
        self.ptAperture = 0.0
        self.ptFocalDistance = 0.0
        self.ptAutoFocus = True
        self.m_totalSamplesAccumulated = 0
        self.m_pushConst = abi.PushConstant()
        self.hdr_integral = None
        self._attached = False
        # adaptive sampling (reference src/renderer_pathtracer.hpp:158-199, .cpp:1326-1374).  The reference defaults to ON for
        # interactive use and its benchmark harness passes --ptAdaptiveSampling 0; this mirror defaults to OFF so that a
        # frame's sample count never depends on timing unless asked for.
        self.ptAdaptiveSampling = False
        # OptiX-style guide image (albedo + camera-space normal of the first hit): set_guide_outputs(True) allocates it, every frame then
        # carries ePtUseOptixDenoiser (reference: the flag follows the denoiser selection, src/renderer_pathtracer.cpp:1547)
        self.ptUseOptixDenoiser = False
        # DLSS variant (set_dlss_guides(True)): one jittered sample per frame, the image replaced, six guide images written.  The
        # frame index restarts on resize (Dlss::notifyReset) and is the frame's frameCount (setupPushConstant :1514-1523).
        self.ptUseDlss = False
        self.m_dlssFrameIndex = 0
        self.m_prevMVP = None          # GltfRenderer::m_prevMVP: the previous frame's viewProjMatrix (src/renderer.cpp:682, 703)
        self.ptPerformanceTarget = 1  # 0 interactive (60 FPS), 1 balanced (30), 2 quality (15), 3 max quality (10)
        self.last_frame_gpu_ms = None  # GPU time of the previous frame's path-trace section (the reference reads its profiler)
        self._held = {}                # what the handle holds, as _EDIT_BYTES sees it

    # -- error plumbing (reference: NVVK_CHECK aborts; here: exceptions carrying b200pt_last_error) --
    def _ck(self, rc, what):
        if rc != 0:
            msg = self._L.b200pt_last_error(self._h)
            raise B200PTError(f"{what} failed ({rc}): {msg.decode() if msg else ''}")

    def registerParameters(self, registry):
        """nvutils::ParameterRegistry analogue: registry is any dict-like; names as the reference CLI."""
        for name in ("ptMaxDepth", "ptSamples", "ptFireflyClamp", "ptTexGradScale", "ptAperture",
                     "ptFocalDistance", "ptAutoFocus", "ptAdaptiveSampling", "ptPerformanceTarget"):
            registry[name] = (self, name)

    # -- BaseRenderer virtuals --------------------------------------------------------------------
    def onAttach(self, resources, profiler=None):
        rc = self._L.b200pt_create(C.byref(self._h), self._device)
        if rc != 0:
            raise B200PTError(f"b200pt_create failed ({rc}): no usable CUDA device {self._device}")
        self._attached = True
        if profiler:
            self._ck(self._L.b200pt_set_profiling(self._h, 1), "b200pt_set_profiling")
        if resources.scene is not None:
            self.onSceneInvalidated(resources)
        if resources.hdr_rgb is not None:
            self.setEnvironment(resources.hdr_rgb)
        self.onResize(None, resources.size, resources)

    def onDetach(self, resources=None):
        if self._attached:
            self._L.b200pt_destroy(self._h)
            self._h = C.c_void_p()
            self._attached = False

    def __del__(self):
        try:
            self.onDetach()
        except Exception:
            pass

    def onSceneInvalidated(self, resources):
        d = resources.scene.desc()
        # SceneOmm::create before SceneRtx's BLAS build (reference renderer: gltf_scene_vk.cpp owns SceneOmm)
        mm, nmm, po, npo, keep = resources.scene.omm_desc()
        self._ck(self._L.b200pt_set_opacity_micromaps(self._h, mm, nmm, po, npo), "b200pt_set_opacity_micromaps")
        self._ck(self._L.b200pt_set_scene(self._h, C.byref(d)), "b200pt_set_scene")
        self._held = {name: state(resources.scene) for name, state in _EDIT_BYTES.items()}

    def set_bvh_builder(self, kind):
        """0: host SAH builder, 1: device LBVH builder (takes effect at the next onSceneInvalidated)"""
        self._ck(self._L.b200pt_set_bvh_builder(self._h, kind), "b200pt_set_bvh_builder")

    def bvh_build_ms(self):
        ms = C.c_double()
        self._ck(self._L.b200pt_bvh_build_ms(self._h, C.byref(ms)), "b200pt_bvh_build_ms")
        return ms.value

    def update_transforms(self, resources):
        """the render nodes of resources.scene moved (same nodes / primitives / materials): refit instead of a rebuild
        (SceneRtx::updateTopLevelAS analogue, b200pt_update_transforms)"""
        scn = resources.scene
        n = len(scn.render_nodes)
        arr = (abi.RenderNode * max(n, 1))()
        for i, rn in enumerate(scn.render_nodes):
            arr[i].objectToWorld[:] = np.asarray(rn["objectToWorld"], np.float32).tolist()
            arr[i].worldToObject[:] = np.asarray(rn["worldToObject"], np.float32).tolist()
            arr[i].materialID = rn["materialID"]
            arr[i].renderPrimID = rn["renderPrimID"]
        self._ck(self._L.b200pt_update_transforms(self._h, arr, n), "b200pt_update_transforms")

    # -- scene edits (GltfRenderer::updateSceneChanges): the handle then renders what onSceneInvalidated of the edited scene would --
    def update_materials(self, resources):
        """the materials / texture infos of resources.scene changed (same material count, same texture images): b200pt_update_materials"""
        scn = resources.scene
        mats = (abi.ShadeMaterial * max(len(scn.materials), 1))(*scn.materials)
        tis = (abi.TextureInfo * max(len(scn.texture_infos), 1))(*scn.texture_infos)
        self._ck(self._L.b200pt_update_materials(self._h, mats, len(scn.materials), tis, len(scn.texture_infos)), "b200pt_update_materials")
        self._held["update_materials"] = _EDIT_BYTES["update_materials"](scn)

    def update_node_materials(self, resources):
        """the render nodes' materialIDs of resources.scene changed (a material variant switch): b200pt_update_node_materials"""
        ids = np.ascontiguousarray([rn["materialID"] for rn in resources.scene.render_nodes] or [0], np.int32)
        self._ck(self._L.b200pt_update_node_materials(self._h, ids.ctypes.data_as(C.POINTER(C.c_int32)), len(resources.scene.render_nodes)),
                 "b200pt_update_node_materials")

    def update_lights(self, resources):
        """the lights of resources.scene changed (their count too): b200pt_update_lights"""
        lights = resources.scene.lights
        arr = (abi.Light * max(len(lights), 1))(*lights)
        self._ck(self._L.b200pt_update_lights(self._h, arr, len(lights)), "b200pt_update_lights")
        self._held["update_lights"] = _EDIT_BYTES["update_lights"](resources.scene)

    def set_node_visibility(self, resources):
        """the render nodes' visibility of resources.scene changed: b200pt_set_node_visibility"""
        vis = np.ascontiguousarray([1 if rn.get("visible", True) else 0 for rn in resources.scene.render_nodes] or [0], np.uint8)
        self._ck(self._L.b200pt_set_node_visibility(self._h, vis.ctypes.data_as(C.POINTER(C.c_uint8)), len(resources.scene.render_nodes)),
                 "b200pt_set_node_visibility")
        self._held["set_node_visibility"] = _EDIT_BYTES["set_node_visibility"](resources.scene)

    def update_scene_changes(self, resources):
        """GltfRenderer::updateSceneChanges for the changes animation.apply_pointers makes to resources.scene: update_materials,
        update_lights and set_node_visibility, each sent only when its bytes differ from what the handle holds.  A visibility change
        rebuilds the trees (DESIGN.md §2), so a channel holding its value must not send it again every frame."""
        for name, state in _EDIT_BYTES.items():
            if self._held.get(name) != state(resources.scene):
                getattr(self, name)(resources)

    def set_animation(self, morph_tasks=(), skin_tasks=()):
        """SceneAnimationVk::createAnimationResources analogue (b200pt_set_animation): uploads the static inputs of the morph /
        skin tasks (vk_gltf_renderer_b200.animation.MorphTask / SkinTask) of the current scene."""
        f32 = lambda a: None if a is None else np.ascontiguousarray(a, np.float32)
        keep = []
        mt = (abi.MorphTask * max(len(morph_tasks), 1))()
        for i, t in enumerate(morph_tasks):
            arrs = [f32(t.base_positions), f32(t.base_normals), f32(t.base_tangents), f32(t.position_deltas), f32(t.normal_deltas), f32(t.tangent_deltas)]
            keep.append(arrs)
            mt[i].renderPrimID, mt[i].vertexCount, mt[i].numTargets = t.render_prim, arrs[0].shape[0], arrs[3].shape[0]
            (mt[i].basePositions, mt[i].baseNormals, mt[i].baseTangents, mt[i].positionDeltas, mt[i].normalDeltas, mt[i].tangentDeltas) = [abi.fptr(a) for a in arrs]
        sk = (abi.SkinTask * max(len(skin_tasks), 1))()
        for i, t in enumerate(skin_tasks):
            arrs = [f32(t.base_positions), f32(t.base_normals), f32(t.base_tangents), f32(t.weights)]
            j = np.ascontiguousarray(t.joints, np.int32)
            keep.append((arrs, j))
            sk[i].renderPrimID, sk[i].vertexCount, sk[i].numJoints = t.render_prim, arrs[0].shape[0], t.num_joints
            sk[i].basePositions, sk[i].baseNormals, sk[i].baseTangents, sk[i].weights = [abi.fptr(a) for a in arrs]
            sk[i].joints = j.ctypes.data_as(C.POINTER(C.c_int32))
        self._ck(self._L.b200pt_set_animation(self._h, mt, len(morph_tasks), sk, len(skin_tasks)), "b200pt_set_animation")
        self._anim = (list(morph_tasks), list(skin_tasks))

    def animate(self, morph_weights=(), joint_matrices=(), normal_matrices=()):
        """one SceneAnimationVk::cmdUpdateAnimation (b200pt_animate): per morph task its target weights, per skin task its joint
        matrices [numJoints, 4, 4] (glm column-major: element [j, c, r]) and normal matrices [numJoints, 3, 3]; vertex arrays,
        shade records and trees are updated on the device."""
        cat = lambda xs, n: np.ascontiguousarray(np.concatenate([np.asarray(x, np.float32).reshape(-1) for x in xs]) if len(xs) else np.zeros(n, np.float32), np.float32)
        w, jm, nm = cat(morph_weights, 1), cat(joint_matrices, 16), cat(normal_matrices, 9)
        self._ck(self._L.b200pt_animate(self._h, w.ctypes.data_as(C.c_void_p), jm.ctypes.data_as(C.c_void_p), nm.ctypes.data_as(C.c_void_p)), "b200pt_animate")

    def set_node_hierarchy(self, parents, mappings, inst_local=None):
        """b200pt_set_node_hierarchy: parents[numNodes] (-1 = root); the BFS levels are derived here the way the reference's
        createGpuBuffers does for its one-dispatch-per-level propagation; mappings: (nodeID, materialID, renderPrimID) per render
        node; inst_local: optional [numRenderNodes, 4, 4] glm-ordered instance matrices."""
        from .animation import topo_levels
        parents = np.ascontiguousarray(parents, np.int32)
        order, offsets = topo_levels(parents)
        mp = (abi.RenderNodeMapping * max(len(mappings), 1))()
        for i, (node, mat, prim) in enumerate(mappings):
            mp[i].nodeID, mp[i].pad0, mp[i].materialID, mp[i].renderPrimID = node, 0, mat, prim
        il = None if inst_local is None else np.ascontiguousarray(inst_local, np.float32)
        g = abi.NodeHierarchy(len(parents), len(offsets) - 1, parents.ctypes.data_as(C.POINTER(C.c_int32)), order.ctypes.data_as(C.POINTER(C.c_int32)),
                              abi.u32ptr(offsets), mp, abi.fptr(il))
        self._ck(self._L.b200pt_set_node_hierarchy(self._h, C.byref(g)), "b200pt_set_node_hierarchy")

    def update_node_matrices(self, local_matrices):
        """b200pt_update_node_matrices: [numNodes, 4, 4] glm-ordered local matrices -> world matrices, render nodes and trees on the device"""
        lm = np.ascontiguousarray(local_matrices, np.float32)
        self._ck(self._L.b200pt_update_node_matrices(self._h, lm.ctypes.data_as(C.c_void_p)), "b200pt_update_node_matrices")

    def setEnvironment(self, rgb):
        rgb = np.ascontiguousarray(rgb, np.float32)
        integral = C.c_float()
        self._ck(self._L.b200pt_set_environment(self._h, rgb.ctypes.data_as(C.c_void_p), rgb.shape[1], rgb.shape[0],
                                                C.byref(integral)), "b200pt_set_environment")
        self.hdr_integral = integral.value

    def onResize(self, cmd, size, resources):
        w, h = size
        if resources.tile and resources.tile[0] == "interleave":
            _, band, world, rank = resources.tile
            self._ck(self._L.b200pt_resize_interleaved(self._h, w, h, band, world, rank), "b200pt_resize_interleaved")
            y0, rows = 0, h // world
        else:
            y0, rows = resources.tile if resources.tile else (0, h)
            self._ck(self._L.b200pt_resize(self._h, w, h, y0, rows), "b200pt_resize")
        self._size = (w, h)
        self._tile = (y0, rows)
        self.m_dlssFrameIndex = 0
        resources.size = (w, h)

    MIN_SAMPLES_PER_PIXEL, MAX_SAMPLES_PER_PIXEL = 1, 100

    def getTargetFrameTimeMs(self):
        return {0: 1000.0 / 60.0, 1: 1000.0 / 30.0, 2: 1000.0 / 15.0, 3: 1000.0 / 10.0}.get(self.ptPerformanceTarget, 1000.0 / 30.0)

    def updateAdaptiveSampling(self, resources):
        """PathTracer::updateAdaptiveSampling (src/renderer_pathtracer.cpp:1326-1374): samples per pixel follow the measured
        GPU time of the path-trace section -- reset to 1 when the accumulation restarts, hands off during the first 5 frames,
        +1 with more than 20 % headroom under the target frame time, -1 when more than 10 % over, clamped to [1, 100]."""
        if not self.ptAdaptiveSampling or self.last_frame_gpu_ms is None and resources.frameCount != 0:
            return
        if resources.frameCount == 0:
            self.ptSamples = self.MIN_SAMPLES_PER_PIXEL
            return
        if resources.frameCount < 5:
            return
        target = self.getTargetFrameTimeMs()
        if self.last_frame_gpu_ms < target * 0.8 and self.ptSamples < self.MAX_SAMPLES_PER_PIXEL:
            self.ptSamples += 1
        elif self.last_frame_gpu_ms > target * 1.1 and self.ptSamples > self.MIN_SAMPLES_PER_PIXEL:
            self.ptSamples -= 1
        self.ptSamples = min(max(self.ptSamples, self.MIN_SAMPLES_PER_PIXEL), self.MAX_SAMPLES_PER_PIXEL)

    def onRender(self, cmd, resources):
        """One frame: updateAdaptiveSampling + setupPushConstant (renderer_pathtracer.cpp:553,1496-1574) + dispatch +
        updateStatistics."""
        w, h = self._size
        s = resources.settings
        self.updateAdaptiveSampling(resources)
        if resources.frameCount == 0:
            self.m_totalSamplesAccumulated = 0
        fi = cam_mod.make_frame_info(resources.camera, w, h, use_hdr=(s.envSystem == 1), env_rotation=s.hdrEnvRotation,
                                     env_intensity=s.hdrEnvIntensity, env_blur=s.hdrBlur,
                                     solid_background=s.useSolidBackground, background=s.solidBackgroundColor,
                                     infinite_plane=s.useInfinitePlane, plane_distance=s.infinitePlaneDistance, plane_color=s.infinitePlaneBaseColor,
                                     plane_metallic=s.infinitePlaneMetallic, plane_roughness=s.infinitePlaneRoughness, shadow_catcher=s.isShadowCatcher,
                                     catcher_darkness=s.shadowCatcherDarkness)
        if self.m_prevMVP is not None:
            fi.prevMVP[:] = self.m_prevMVP
        self.m_prevMVP = list(fi.viewProjMatrix)
        num_samples = 1 if self.ptUseDlss else self.ptSamples
        pc = cam_mod.make_push_constant(resources.camera, h, frame_count=resources.frameCount,
                                        total_samples=self.m_totalSamplesAccumulated, num_samples=num_samples,
                                        max_depth=self.ptMaxDepth, firefly_clamp=self.ptFireflyClamp,
                                        tex_grad_scale=self.ptTexGradScale, aperture=self.ptAperture,
                                        focal_distance=None if self.ptAutoFocus else self.ptFocalDistance)
        if self.ptUseDlss:
            # setupPushConstant :1514-1523, 1543: the Halton index is the frameCount; ePtFirstFrame still follows resources.frameCount
            self.m_dlssFrameIndex += 1
            pc.frameCount = self.m_dlssFrameIndex
            fi.jitter[:] = list(cam_mod.dlss_jitter(self.m_dlssFrameIndex))
            pc.flags |= abi.PT_USE_DLSS
        if self.ptUseOptixDenoiser:
            pc.flags |= abi.PT_USE_OPTIX_DENOISER   # setupPushConstant :1547
        self.m_pushConst = pc
        self._ck(self._L.b200pt_render_frame(self._h, C.byref(fi), C.byref(pc)), "b200pt_render_frame")
        self.m_totalSamplesAccumulated += num_samples

    # -- C-ABI passthroughs -------------------------------------------------------------------------
    def render_frame_raw(self, fi, pc):
        self._ck(self._L.b200pt_render_frame(self._h, C.byref(fi), C.byref(pc)), "b200pt_render_frame")

    def synchronize(self):
        self._ck(self._L.b200pt_synchronize(self._h), "b200pt_synchronize")

    def read_accum(self):
        w, _ = self._size
        rows = self._tile[1]
        out = np.empty((rows, w, 4), np.float32)
        self._ck(self._L.b200pt_read_accum(self._h, out.ctypes.data_as(C.c_void_p), out.size), "b200pt_read_accum")
        return out

    @staticmethod
    def make_tonemapper(method=0, isActive=1, exposure=1.0, brightness=1.0, contrast=1.0, saturation=1.0, vignette=0.0, autoExposure=0):
        """shaderio::TonemapperData defaults (filmic, everything neutral); the reference's Resources turns autoExposure on"""
        return abi.Tonemapper(method, isActive, exposure, brightness, contrast, saturation, vignette, autoExposure)

    def tonemap(self, tm=None):
        """GltfRenderer::tonemap (src/renderer.cpp:992-1054): eImgRendered -> eImgTonemapped.  Returns (RGBA8 [rows, width, 4],
        exposure factor used)."""
        tm = tm or self.make_tonemapper()
        w, _ = self._size
        rows = self._tile[1]
        out = np.empty((rows, w, 4), np.uint8)
        ex = C.c_float()
        self._ck(self._L.b200pt_tonemap(self._h, C.byref(tm), out.ctypes.data_as(C.c_void_p), out.size, C.byref(ex)), "b200pt_tonemap")
        return out, ex.value

    def tonemap_image(self, tm, dev_rgba32f, width, height, dev_rgba8):
        """device RGBA32F image (e.g. the gathered multi-GPU frame) -> device RGBA8; returns the exposure factor used"""
        ex = C.c_float()
        self._ck(self._L.b200pt_tonemap_image(self._h, C.byref(tm), C.c_void_p(dev_rgba32f), width, height, C.c_void_p(dev_rgba8), C.byref(ex)), "b200pt_tonemap_image")
        return ex.value

    def set_guide_outputs(self, enable=True):
        """b200pt_set_guide_outputs: the path pools carry the first-hit guides, frames write OutputImage::eOptixAlbedoNormal"""
        self._ck(self._L.b200pt_set_guide_outputs(self._h, 1 if enable else 0), "b200pt_set_guide_outputs")
        self.ptUseOptixDenoiser = bool(enable)

    def read_guide(self):
        """eOptixAlbedoNormal of the newest frame: (albedo float32 [rows, W, 3], compressed camera-space normal uint32 [rows, W])"""
        w, _ = self._size
        rows = self._tile[1]
        out = np.empty((rows, w, 4), np.float32)
        self._ck(self._L.b200pt_read_guide(self._h, out.ctypes.data_as(C.c_void_p), out.size), "b200pt_read_guide")
        return out[..., :3].copy(), out[..., 3].copy().view(np.uint32)

    def set_dlss_guides(self, enable=True):
        """b200pt_set_dlss_guides: the path pools carry the DLSS scratch; every frame then runs the DLSS variant"""
        self._ck(self._L.b200pt_set_dlss_guides(self._h, 1 if enable else 0), "b200pt_set_dlss_guides")
        self.ptUseDlss = bool(enable)

    DLSS_PLANES = (("albedo", np.uint8, 4), ("spec_albedo", np.float16, 4), ("normal_roughness", np.float16, 4),
                   ("motion", np.float16, 2), ("depth", np.float16, 1), ("spec_hit_dist", np.float16, 1))

    def read_dlss_guides(self):
        """the six DLSS guide images of the newest frame: albedo uint8 [rows, W, 4] (RGBA8 UNORM), spec_albedo and
        normal_roughness float16 [rows, W, 4], motion float16 [rows, W, 2] (pixels), depth and spec_hit_dist float16 [rows, W]"""
        w, _ = self._size
        rows = self._tile[1]
        out, g = {}, abi.DlssGuides()
        for name, dt, ch in self.DLSS_PLANES:
            a = np.empty((rows, w, ch) if ch > 1 else (rows, w), dt)
            out[name] = a
            setattr(g, name, a.ctypes.data)
            setattr(g, name + "_bytes", a.nbytes)
        self._ck(self._L.b200pt_read_dlss_guides(self._h, C.byref(g)), "b200pt_read_dlss_guides")
        return out

    def read_selection(self):
        """gBuffers[eImgSelection] (object id per pixel, render node + 1, 0 = miss) and the NDC depth image, as the first
        frame of the current accumulation wrote them (gltf_pathtrace.slang:604-616)."""
        w, _ = self._size
        rows = self._tile[1]
        ids = np.empty((rows, w), np.uint32)
        depth = np.empty((rows, w), np.float32)
        self._ck(self._L.b200pt_read_selection(self._h, ids.ctypes.data_as(C.c_void_p), depth.ctypes.data_as(C.c_void_p), ids.size), "b200pt_read_selection")
        return ids, depth

    def read_accum_async(self, host_ptr, num_floats, slot):
        """enqueue a copy of the image into (pinned) host memory; wait_read(slot) completes it."""
        self._ck(self._L.b200pt_read_accum_async(self._h, host_ptr, num_floats, slot), "b200pt_read_accum_async")

    def wait_read(self, slot):
        self._ck(self._L.b200pt_wait_read(self._h, slot), "b200pt_wait_read")

    def set_frames_in_flight(self, n):
        self._ck(self._L.b200pt_set_frames_in_flight(self._h, n), "b200pt_set_frames_in_flight")

    def set_frame_batch(self, n):
        """collect up to n consecutive frames of a static camera into one wavefront (include/b200pt.h)"""
        self._ck(self._L.b200pt_set_frame_batch(self._h, n), "b200pt_set_frame_batch")

    def flush(self):
        self._ck(self._L.b200pt_flush(self._h), "b200pt_flush")

    def set_views(self, n):
        """render n camera poses of one frame as one wavefront, each into its own images (include/b200pt.h); clears the images"""
        self._ck(self._L.b200pt_set_views(self._h, n), "b200pt_set_views")
        self._views = n

    def render_views(self, fis, pc):
        """one frame of every view: fis is a sequence of FrameInfo that differ only in their pose (camera.view_frame_infos)"""
        arr = fis if isinstance(fis, C.Array) else (abi.FrameInfo * len(fis))(*fis)
        self._ck(self._L.b200pt_render_views(self._h, arr, len(arr), C.byref(pc)), "b200pt_render_views")

    def read_views(self):
        """every view's images: RGBA32F [V, rows, W, 4], object ids uint32 [V, rows, W] and NDC depth float32 [V, rows, W]"""
        w, _ = self._size
        rows = self._tile[1]
        v = getattr(self, "_views", 1)
        rgba = np.empty((v, rows, w, 4), np.float32)
        ids = np.empty((v, rows, w), np.uint32)
        depth = np.empty((v, rows, w), np.float32)
        for k in range(v):
            self._ck(self._L.b200pt_read_views(self._h, k, rgba[k].ctypes.data_as(C.c_void_p), ids[k].ctypes.data_as(C.c_void_p),
                                               depth[k].ctypes.data_as(C.c_void_p), rows * w), "b200pt_read_views")
        return rgba, ids, depth

    def views_device_ptrs(self, view):
        """device pointers of one view's RGBA32F, object-id and depth images"""
        rgba, ids, depth = C.c_void_p(), C.c_void_p(), C.c_void_p()
        self._ck(self._L.b200pt_get_views_device(self._h, view, C.byref(rgba), C.byref(ids), C.byref(depth)), "b200pt_get_views_device")
        return rgba.value, ids.value, depth.value

    def set_convergence(self, threshold, floor=1e-3, min_frames=16, interval=8):
        """stop each pixel of the next accumulation once its relative error e <= threshold (include/b200pt.h, DESIGN.md §2
        "Convergence"); threshold 0 turns it off.  Takes effect at the next frame with frameCount 0."""
        c = abi.Convergence(threshold, floor, min_frames, interval)
        self._ck(self._L.b200pt_set_convergence(self._h, C.byref(c)), "b200pt_set_convergence")
        self._convergence = c if threshold != 0 else None

    def read_convergence(self):
        """(stop frame uint32 [rows, W] (0 = active), relative error float32 [rows, W], active pixels) of the current accumulation"""
        w, _ = self._size
        rows = self._tile[1]
        stop = np.empty((rows, w), np.uint32)
        err = np.empty((rows, w), np.float32)
        active = C.c_uint32()
        self._ck(self._L.b200pt_read_convergence(self._h, stop.ctypes.data_as(C.c_void_p), err.ctypes.data_as(C.c_void_p), stop.size, C.byref(active)),
                 "b200pt_read_convergence")
        return stop, err, active.value

    def accum_device_ptr(self):
        p, n = C.c_void_p(), C.c_size_t()
        self._ck(self._L.b200pt_get_accum_device(self._h, C.byref(p), C.byref(n)), "b200pt_get_accum_device")
        return p.value, n.value

    def set_accum_device(self, ptr, num_floats):
        self._ck(self._L.b200pt_set_accum_device(self._h, C.c_void_p(ptr), num_floats), "b200pt_set_accum_device")

    def stream(self):
        return self._L.b200pt_stream(self._h)

    def stats(self):
        st = abi.Stats()
        self._ck(self._L.b200pt_get_stats(self._h, C.byref(st)), "b200pt_get_stats")
        return {n: getattr(st, n) for n, _ in abi.Stats._fields_}

    def reset_stats(self):
        self._ck(self._L.b200pt_reset_stats(self._h), "b200pt_reset_stats")

    def set_profiling(self, on):
        self._ck(self._L.b200pt_set_profiling(self._h, 1 if on else 0), "b200pt_set_profiling")

    def bvh_info(self):
        nb, tb, nn, nt = C.c_uint64(), C.c_uint64(), C.c_uint32(), C.c_uint32()
        self._ck(self._L.b200pt_bvh_info(self._h, C.byref(nb), C.byref(tb), C.byref(nn), C.byref(nt)), "b200pt_bvh_info")
        return dict(node_bytes=nb.value, tri_bytes=tb.value, num_nodes=nn.value, num_tris=nt.value)

    # ray-level entry points take device pointers (ints), e.g. torch tensors' data_ptr()
    def trace_closest(self, rays_ptr, n, hits_ptr, seeds_ptr=None):
        self._ck(self._L.b200pt_trace_closest(self._h, C.c_void_p(rays_ptr), n, C.c_void_p(hits_ptr),
                                              C.c_void_p(seeds_ptr) if seeds_ptr else None), "b200pt_trace_closest")

    def trace_shadow(self, rays_ptr, n, out_ptr, seeds_ptr=None):
        self._ck(self._L.b200pt_trace_shadow(self._h, C.c_void_p(rays_ptr), n, C.c_void_p(out_ptr),
                                             C.c_void_p(seeds_ptr) if seeds_ptr else None), "b200pt_trace_shadow")

    def bsdf_eval(self, in_ptr, n, out_ptr):
        self._ck(self._L.b200pt_bsdf_eval(self._h, C.c_void_p(in_ptr), n, C.c_void_p(out_ptr)), "b200pt_bsdf_eval")

    def bsdf_sample(self, in_ptr, n, out_ptr):
        self._ck(self._L.b200pt_bsdf_sample(self._h, C.c_void_p(in_ptr), n, C.c_void_p(out_ptr)), "b200pt_bsdf_sample")

    def texture_lookup(self, in_ptr, n, out_ptr):
        """n texture lookups (records of tex_io, device pointers) against the attached scene: rgba, 4 floats each"""
        self._ck(self._L.b200pt_texture_lookup(self._h, C.c_void_p(in_ptr), n, C.c_void_p(out_ptr)), "b200pt_texture_lookup")

    def shade_state(self, in_ptr, n, out_ptr, seeds_ptr=None):
        """n rays (records of shade_io, device pointers) through the closest-hit walk, the hit fetch and evaluateMaterial of the
        attached scene's shade variant: 96 floats each"""
        self._ck(self._L.b200pt_shade_state(self._h, C.c_void_p(in_ptr), n, C.c_void_p(out_ptr), C.c_void_p(seeds_ptr) if seeds_ptr else None),
                 "b200pt_shade_state")


def render_headless(resources, frames, *, pt=None, device=0, until_converged=False, **pt_params):
    """The reference's headless loop (src/main.cpp:133-136 + nvapp frame loop, SURVEY.md §3.1):
    frameCount runs 0..frames-1, each frame adds ptSamples spp.  Returns (PathTracer, accum RGBA32F).
    until_converged: with pt.set_convergence on, the loop also ends after the first checkpoint at which no pixel is active (the
    count is read at checkpoints only, since the read synchronises); resources.frameCount is then the last frame rendered."""
    own = pt is None
    if own:
        pt = PathTracer(device)
        for k, v in pt_params.items():
            setattr(pt, k, v)
        pt.onAttach(resources)
    conv = getattr(pt, "_convergence", None) if until_converged else None
    resources.frameCount = -1
    # (the headless run raises maxFrames to the frame count: BenchmarkController::alignMaxFramesForHeadless, so no cap applies)
    for _ in range(frames):
        resources.frameCount += 1
        pt.onRender(None, resources)
        if conv is not None and (resources.frameCount + 1) % conv.interval == 0 and pt.read_convergence()[2] == 0:
            break
    img = pt.read_accum()
    return pt, img
