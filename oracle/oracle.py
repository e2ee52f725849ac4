"""ctypes binding of the CPU oracle (oracle/liboracle_pt.so).   *** TEST INFRASTRUCTURE ***

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
import this module.  The product package (vk_gltf_renderer_b200) never does.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "liboracle_pt.so")


def build(force=False):
    src = [os.path.join(_HERE, f) for f in ("pt_oracle.cpp", "bsdf.h", "vecmath.h")]
    if force or not os.path.exists(_LIB_PATH) or any(
            os.path.exists(s) and os.path.getmtime(s) > os.path.getmtime(_LIB_PATH) for s in src):
        subprocess.check_call(["make", "-C", _HERE, "-s"])
    return _LIB_PATH


_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH):
            build()
        L = C.CDLL(_LIB_PATH)
        L.oracle_create.restype = C.c_void_p
        L.oracle_destroy.argtypes = [C.c_void_p]
        L.oracle_set_scene.argtypes = [C.c_void_p, C.c_void_p]
        L.oracle_set_opacity_micromaps.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32]
        L.oracle_set_environment.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]
        L.oracle_get_environment.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.oracle_render_frame.argtypes = [C.c_void_p] * 9 + [C.c_int] * 3
        L.oracle_trace_closest.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
        L.oracle_trace_shadow.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
        L.oracle_trace_closest_mt.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_int]
        L.oracle_bsdf_eval.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p]
        L.oracle_bsdf_sample.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p]
        L.oracle_bsdf_sample_simple.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p]
        L.oracle_bsdf_eval_simple.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p]
        L.oracle_dlss_env_brdf_approx2.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p]
        L.oracle_hg_sample.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p]
        L.oracle_hg_pdf.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p]
        L.oracle_ssa.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p]
        L.oracle_dlss_motion_vector.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
        L.oracle_get_stats.argtypes = [C.c_void_p, C.c_void_p]
        L.oracle_reset_stats.argtypes = [C.c_void_p]
        L.oracle_num_tris.argtypes = [C.c_void_p]
        L.oracle_xxhash32.restype = C.c_uint32
        L.oracle_xxhash32.argtypes = [C.c_uint32] * 3
        L.oracle_rand.restype = C.c_float
        L.oracle_rand.argtypes = [C.c_void_p]
        L.oracle_safe_offset_ray.argtypes = [C.c_void_p] * 3
        L.oracle_sample_texture.argtypes = [C.c_void_p, C.c_int, C.c_float, C.c_float, C.c_float, C.c_void_p]
        L.oracle_texture_lookup.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p]
        L.oracle_shade_state.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


class Oracle:
    # the DLSS guide planes (name, dtype, channels), in the order of oracle_render_frame's dlssPlanes
    DLSS_PLANES = (("albedo", np.uint8, 4), ("spec_albedo", np.float16, 4), ("normal_roughness", np.float16, 4),
                   ("motion", np.float16, 2), ("depth", np.float16, 1), ("spec_hit_dist", np.float16, 1))

    def __init__(self):
        self.L = lib()
        self.h = C.c_void_p(self.L.oracle_create())
        self._scene = None
        self.env_size = None

    def close(self):
        if self.h:
            self.L.oracle_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_scene(self, scene):
        self._scene = scene
        d = scene.desc()
        rc = self.L.oracle_set_scene(self.h, C.byref(d))
        if rc:
            raise RuntimeError(f"oracle_set_scene failed: {rc}")
        mm, nmm, po, npo, keep = scene.omm_desc()
        if self.L.oracle_set_opacity_micromaps(self.h, C.byref(mm), nmm, C.byref(po), npo):
            raise RuntimeError("oracle_set_opacity_micromaps failed")

    def set_environment(self, rgb):
        rgb = np.ascontiguousarray(rgb, np.float32)
        h, w = rgb.shape[:2]
        integral = C.c_float()
        self.L.oracle_set_environment(self.h, _p(rgb), w, h, C.byref(integral))
        self.env_size = (w, h)
        return integral.value

    def get_environment(self):
        w, h = self.env_size
        rgba = np.empty((h, w, 4), np.float32)
        alias = np.empty(h * w, np.uint32)
        q = np.empty(h * w, np.float32)
        self.L.oracle_get_environment(self.h, _p(rgba), _p(alias), _p(q))
        return rgba, alias, q

    def render_frame(self, fi, pc, accum, y0=0, rows=None, threads=None, object_id=None, ndc_depth=None, guide=None):
        """accum: float32 [rows, W, 4], updated in place (running mean like processPixel).  object_id (uint32 [rows, W]) /
        ndc_depth (float32 [rows, W]), if given, receive the frame-0 outputs (selection ray id, NDC depth of the first hit);
        guide (float32 [rows, W, 4]) the eOptixAlbedoNormal image of a frame whose push constants carry ePtUseOptixDenoiser.
        A DLSS frame (pc carries PT_USE_DLSS) raises ValueError: it writes guide planes, so it goes through render_frame_dlss."""
        self._render_frame(fi, pc, accum, y0, rows, threads, object_id, ndc_depth, guide)

    def render_frame_dlss(self, fi, pc, accum, prev_object_to_world=None, y0=0, rows=None, threads=None, object_id=None, ndc_depth=None,
                          guide=None):
        """A frame of the DLSS variant (pc carries PT_USE_DLSS): accum (float32 [rows, W, 4]) is replaced; returns the six guide
        planes as a dict of arrays shaped like PathTracer.read_dlss_guides().  prev_object_to_world: float32 [numRenderNodes, 16]
        (the previous frame's objectToWorld, glm order) or None for camera-only motion.  A frame the variant refuses (no PT_USE_DLSS,
        numSamples != 1) raises ValueError."""
        rows = accum.shape[0] if rows is None else rows
        w = accum.shape[1]
        planes = {name: np.zeros((rows, w, ch) if ch > 1 else (rows, w), dt) for name, dt, ch in self.DLSS_PLANES}
        prev = None if prev_object_to_world is None else np.ascontiguousarray(prev_object_to_world, np.float32)
        self._render_frame(fi, pc, accum, y0, rows, threads, object_id, ndc_depth, guide, prev, planes)
        return planes

    def _render_frame(self, fi, pc, accum, y0, rows, threads, object_id, ndc_depth, guide, prev=None, planes=None):
        rows = accum.shape[0] if rows is None else rows
        threads = threads or os.cpu_count() or 1
        ptrs = None if planes is None else (C.c_void_p * 6)(*[planes[name].ctypes.data for name, _, _ in self.DLSS_PLANES])
        rc = self.L.oracle_render_frame(self.h, C.byref(fi), C.byref(pc), _p(accum), _p(object_id), _p(ndc_depth), _p(guide), _p(prev), ptrs,
                                        y0, rows, threads)
        if rc == -1:   # B200PT_E_INVALID
            raise ValueError("oracle_render_frame: a DLSS frame (PT_USE_DLSS) needs numSamples == 1 and the guide planes of render_frame_dlss; "
                             "a plain frame takes no planes")
        if rc:
            raise RuntimeError(f"oracle_render_frame failed: {rc}")

    def trace_closest(self, rays, seeds=None, threads=1):
        rays = np.ascontiguousarray(rays, np.float32).reshape(-1, 8)
        hits = np.empty((len(rays), 6), np.float32)
        if threads > 1 and seeds is None:
            self.L.oracle_trace_closest_mt(self.h, _p(rays), len(rays), _p(hits), threads)
        else:
            self.L.oracle_trace_closest(self.h, _p(rays), len(rays), _p(hits), _p(seeds))
        return hits

    def trace_shadow(self, rays, seeds=None):
        rays = np.ascontiguousarray(rays, np.float32).reshape(-1, 8)
        out = np.empty((len(rays), 3), np.float32)
        self.L.oracle_trace_shadow(self.h, _p(rays), len(rays), _p(out), _p(seeds))
        return out

    def bsdf_eval(self, packed):
        packed = np.ascontiguousarray(packed, np.float32).reshape(-1, 48)
        out = np.empty((len(packed), 8), np.float32)
        self.L.oracle_bsdf_eval(_p(packed), len(packed), _p(out))
        return out

    def bsdf_sample(self, packed):
        packed = np.ascontiguousarray(packed, np.float32).reshape(-1, 48)
        out = np.empty((len(packed), 8), np.float32)
        self.L.oracle_bsdf_sample(_p(packed), len(packed), _p(out))
        return out

    def bsdf_sample_simple(self, packed):
        """bsdfSampleSimple (the shadow catcher's continuation BSDF) on the records of bsdf_io: k2, bsdf_over_pdf, pdf, event"""
        packed = np.ascontiguousarray(packed, np.float32).reshape(-1, 48)
        out = np.empty((len(packed), 8), np.float32)
        self.L.oracle_bsdf_sample_simple(_p(packed), len(packed), _p(out))
        return out

    def bsdf_eval_simple(self, packed):
        """bsdfEvaluateSimple on the records of bsdf_io: bsdf_diffuse, bsdf_glossy, pdf, 0"""
        packed = np.ascontiguousarray(packed, np.float32).reshape(-1, 48)
        out = np.empty((len(packed), 8), np.float32)
        self.L.oracle_bsdf_eval_simple(_p(packed), len(packed), _p(out))
        return out

    def stats(self):
        a = np.zeros(6, np.uint64)
        self.L.oracle_get_stats(self.h, _p(a))
        return dict(closestRays=int(a[0]), shadowRays=int(a[1]), shadedHits=int(a[2]), paths=int(a[3]),
                    nodesVisited=int(a[4]), trisTested=int(a[5]))

    def reset_stats(self):
        self.L.oracle_reset_stats(self.h)

    def num_tris(self):
        return self.L.oracle_num_tris(self.h)

    def sample_texture(self, tex, u, v, g=0.0):
        out = np.zeros(4, np.float32)
        self.L.oracle_sample_texture(self.h, tex, u, v, g, _p(out))
        return out

    def texture_lookup(self, records):
        """getTexture / sampleLevel0 on the records of vk_gltf_renderer_b200.tex_io: rgba float32 [n, 4]"""
        records = np.ascontiguousarray(records, np.float32).reshape(-1, 8)
        out = np.empty((len(records), 4), np.float32)
        if self.L.oracle_texture_lookup(self.h, _p(records), len(records), _p(out)):
            raise ValueError("oracle_texture_lookup: a record has a texture-info slot outside the scene or a mode other than 0 / 1")
        return out

    def shade_state(self, records, seeds=None):
        """closest hit, getHitState, texture gradient and evaluateMaterial on the records of vk_gltf_renderer_b200.shade_io:
        float32 [n, 96]; seeds (uint32 [n], the any-hit draws) are advanced in place"""
        records = np.ascontiguousarray(records, np.float32).reshape(-1, 16)
        out = np.empty((len(records), 96), np.float32)
        self.L.oracle_shade_state(self.h, _p(records), len(records), _p(out), _p(seeds))
        return out

    def hg_sample(self, records):
        """sampleHenyeyGreenstein on float32 [n, 6] records (xi.x, xi.y, g, wi xyz) -> directions [n, 3]"""
        records = np.ascontiguousarray(records, np.float32).reshape(-1, 6)
        out = np.empty((len(records), 3), np.float32)
        self.L.oracle_hg_sample(_p(records), len(records), _p(out))
        return out

    def hg_pdf(self, records):
        """henyeyGreensteinPdf on float32 [n, 2] records (cos theta, g) -> [n]"""
        records = np.ascontiguousarray(records, np.float32).reshape(-1, 2)
        out = np.empty(len(records), np.float32)
        self.L.oracle_hg_pdf(_p(records), len(records), _p(out))
        return out

    def ssa(self, rho):
        """multiToSingleScatterAlbedo of float32 rho [n] (one channel) -> [n]"""
        rho = np.ascontiguousarray(rho, np.float32).reshape(-1)
        out = np.empty(len(rho), np.float32)
        self.L.oracle_ssa(_p(rho), len(rho), _p(out))
        return out

    def env_brdf_approx2(self, records):
        """EnvBRDFApprox2 on float32 [n, 5] records (specular colour xyz, alpha, NoV) -> [n, 3]"""
        records = np.ascontiguousarray(records, np.float32).reshape(-1, 5)
        out = np.empty((len(records), 3), np.float32)
        self.L.oracle_dlss_env_brdf_approx2(_p(records), len(records), _p(out))
        return out

    def motion_vector(self, records, prev_mvp, curr_mvp):
        """calculateMotionVector on float32 [n, 10] records (current xyzw, previous xyzw, resolution xy) -> pixel motion [n, 2]"""
        records = np.ascontiguousarray(records, np.float32).reshape(-1, 10)
        out = np.empty((len(records), 2), np.float32)
        self.L.oracle_dlss_motion_vector(_p(records), len(records), _p(np.ascontiguousarray(prev_mvp, np.float32)),
                                    _p(np.ascontiguousarray(curr_mvp, np.float32)), _p(out))
        return out


def render(oracle, cam, width, height, frames, *, max_depth=5, num_samples=1, threads=None, **fi_kw):
    """Headless loop: `frames` frames of `num_samples` spp, like the reference's --frames/--ptSamples
    (src/renderer.cpp:1959-1977, src/renderer_pathtracer.cpp:1377-1402)."""
    from vk_gltf_renderer_b200 import camera as camm
    accum = np.zeros((height, width, 4), np.float32)
    fi = camm.make_frame_info(cam, width, height, **fi_kw)
    total = 0
    for f in range(frames):
        pc = camm.make_push_constant(cam, height, frame_count=f, total_samples=total, num_samples=num_samples,
                                     max_depth=max_depth)
        oracle.render_frame(fi, pc, accum, threads=threads)
        total += num_samples
    return accum
