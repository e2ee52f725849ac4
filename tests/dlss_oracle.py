"""ctypes binding of the DLSS variant of the CPU oracle (tests/dlss_oracle.cpp).   *** TEST INFRASTRUCTURE ***

The library is compiled on first use into the temporary directory (keyed by the sources, so an edited oracle is rebuilt) with the
oracle's own flags; it contains the whole oracle, so a DlssOracle loads scenes and environments like oracle.oracle.Oracle and adds
the DLSS frame and the DLSS arithmetic entry points.
"""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from oracle import oracle as O

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_SOURCES = [os.path.join(_HERE, "dlss_oracle.cpp")] + [os.path.join(_ROOT, "oracle", f) for f in ("pt_oracle.cpp", "bsdf.h", "vecmath.h")] + \
    [os.path.join(_ROOT, "include", "b200pt.h")]
# oracle/Makefile's flags: scalar fp32 without implicit FMA
_CXXFLAGS = ["-O2", "-march=x86-64-v3", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-std=c++17", "-Wall", "-Wextra", "-pthread", "-shared"]
_lib = None


def build():
    h = hashlib.sha256()
    for s in _SOURCES:
        with open(s, "rb") as f:
            h.update(f.read())
    path = os.path.join(tempfile.gettempdir(), "b200pt_oracle_dlss_%s.so" % h.hexdigest()[:16])
    if not os.path.exists(path):
        tmp = "%s.%d.tmp" % (path, os.getpid())
        subprocess.check_call(["g++"] + _CXXFLAGS + ["-o", tmp, _SOURCES[0]])
        os.replace(tmp, path)
    return path


def lib():
    global _lib
    if _lib is None:
        base = O.lib()
        L = C.CDLL(build())
        for name, f in list(base.__dict__.items()):   # the oracle's entry points, with the argument types oracle.py declares
            if name.startswith("oracle_") and hasattr(f, "argtypes"):
                g = getattr(L, name)
                g.argtypes, g.restype = f.argtypes, f.restype
        L.oracle_render_frame_dlss.argtypes = [C.c_void_p] * 9 + [C.c_int] * 3
        L.oracle_env_brdf_approx2.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p]
        L.oracle_motion_vector.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
        _lib = L
    return _lib


_p = O._p


class DlssOracle(O.Oracle):
    DLSS_PLANES = (("albedo", np.uint8, 4), ("spec_albedo", np.float16, 4), ("normal_roughness", np.float16, 4),
                   ("motion", np.float16, 2), ("depth", np.float16, 1), ("spec_hit_dist", np.float16, 1))

    def __init__(self):
        self.L = lib()
        self.h = C.c_void_p(self.L.oracle_create())
        self._scene = None
        self.env_size = None

    def render_frame_dlss(self, fi, pc, accum, prev_object_to_world=None, y0=0, rows=None, threads=None, object_id=None, ndc_depth=None,
                          guide=None):
        """A frame of the DLSS variant (pc carries PT_USE_DLSS): accum (float32 [rows, W, 4]) is replaced; returns the six guide
        planes as a dict of arrays shaped like PathTracer.read_dlss_guides().  prev_object_to_world: float32 [numRenderNodes, 16]
        (the previous frame's objectToWorld, glm order) or None for camera-only motion.  A frame the variant refuses (no PT_USE_DLSS,
        numSamples != 1) raises ValueError."""
        rows = accum.shape[0] if rows is None else rows
        w = accum.shape[1]
        threads = threads or os.cpu_count() or 1
        planes = {name: np.zeros((rows, w, ch) if ch > 1 else (rows, w), dt) for name, dt, ch in self.DLSS_PLANES}
        ptrs = (C.c_void_p * 6)(*[planes[name].ctypes.data for name, _, _ in self.DLSS_PLANES])
        prev = None if prev_object_to_world is None else np.ascontiguousarray(prev_object_to_world, np.float32)
        rc = self.L.oracle_render_frame_dlss(self.h, C.byref(fi), C.byref(pc), _p(accum), _p(object_id), _p(ndc_depth), _p(guide), _p(prev), ptrs,
                                             y0, rows, threads)
        if rc == -1:   # B200PT_E_INVALID
            raise ValueError("oracle_render_frame_dlss: needs PT_USE_DLSS and numSamples == 1")
        if rc:
            raise RuntimeError(f"oracle_render_frame_dlss failed: {rc}")
        return planes

    def env_brdf_approx2(self, records):
        """EnvBRDFApprox2 on float32 [n, 5] records (specular colour xyz, alpha, NoV) -> [n, 3]"""
        records = np.ascontiguousarray(records, np.float32).reshape(-1, 5)
        out = np.empty((len(records), 3), np.float32)
        self.L.oracle_env_brdf_approx2(_p(records), len(records), _p(out))
        return out

    def motion_vector(self, records, prev_mvp, curr_mvp):
        """calculateMotionVector on float32 [n, 10] records (current xyzw, previous xyzw, resolution xy) -> pixel motion [n, 2]"""
        records = np.ascontiguousarray(records, np.float32).reshape(-1, 10)
        out = np.empty((len(records), 2), np.float32)
        self.L.oracle_motion_vector(_p(records), len(records), _p(np.ascontiguousarray(prev_mvp, np.float32)),
                                    _p(np.ascontiguousarray(curr_mvp, np.float32)), _p(out))
        return out
