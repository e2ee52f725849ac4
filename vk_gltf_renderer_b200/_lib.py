"""Loader for the CUDA library (libb200pt.so) behind include/b200pt.h.

There is NO CPU fallback: if the library is missing or fails to load this raises.
"""
import ctypes as C
import os
import subprocess

from . import abi

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libb200pt.so")

# every symbol include/b200pt.h declares
EXPORTS = [
    "b200pt_create", "b200pt_destroy", "b200pt_abi_version", "b200pt_last_error", "b200pt_set_scene",
    "b200pt_set_environment", "b200pt_resize", "b200pt_resize_interleaved", "b200pt_read_accum_async", "b200pt_wait_read", "b200pt_set_frames_in_flight", "b200pt_render_frame", "b200pt_synchronize",
    "b200pt_get_accum_device", "b200pt_read_accum", "b200pt_set_accum_device", "b200pt_stream",
    "b200pt_get_stats", "b200pt_reset_stats", "b200pt_set_profiling", "b200pt_trace_closest",
    "b200pt_trace_shadow", "b200pt_bvh_info", "b200pt_bsdf_eval", "b200pt_bsdf_sample", "b200pt_texture_lookup", "b200pt_shade_state",
    "b200pt_read_selection", "b200pt_get_selection_device", "b200pt_set_frame_batch", "b200pt_flush", "b200pt_update_transforms", "b200pt_set_bvh_builder", "b200pt_bvh_build_ms",
    "b200pt_set_opacity_micromaps", "b200pt_set_animation", "b200pt_animate", "b200pt_set_node_hierarchy", "b200pt_update_node_matrices", "b200pt_tonemap", "b200pt_tonemap_image", "b200pt_get_tonemapped_device", "b200pt_set_guide_outputs", "b200pt_read_guide", "b200pt_get_guide_device",
    "b200pt_set_dlss_guides", "b200pt_read_dlss_guides", "b200pt_get_dlss_guides_device",
    "b200pt_update_materials", "b200pt_update_node_materials", "b200pt_update_lights", "b200pt_set_node_visibility",
]


def build(verbose=False):
    """Compile libb200pt.so for sm_90a in-tree (nvcc cross-compiles without a GPU)."""
    subprocess.check_call(["make", "-C", os.path.join(_HERE, "csrc"), "-s"],
                          stdout=None if verbose else subprocess.DEVNULL)
    return LIB_PATH


COUNT_LIB_PATH = os.path.join(_HERE, "libb200pt_count.so")
_libs = {}


def lib(count_traversal=False):
    """count_traversal=True loads the variant compiled with -DB200PT_COUNT_TRAVERSAL (per-ray node /
    triangle counters for the roofline model; never used for timing)."""
    path = COUNT_LIB_PATH if count_traversal else os.environ.get("B200PT_LIB", LIB_PATH)  # B200PT_LIB: tuning builds
    if path in _libs:
        return _libs[path]
    if not os.path.exists(path):
        raise RuntimeError(f"{path} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                           "(the CUDA path is the product; there is no fallback)")
    L = C.CDLL(path)
    vp, i32, u32, f32p = C.c_void_p, C.c_int, C.c_uint32, C.c_void_p
    L.b200pt_create.argtypes = [C.POINTER(vp), i32]
    L.b200pt_destroy.argtypes = [vp]
    L.b200pt_destroy.restype = None
    L.b200pt_abi_version.restype = i32
    L.b200pt_last_error.argtypes = [vp]
    L.b200pt_last_error.restype = C.c_char_p
    L.b200pt_set_scene.argtypes = [vp, C.POINTER(abi.SceneDesc)]
    L.b200pt_set_opacity_micromaps.argtypes = [vp, C.POINTER(abi.Micromap), u32, C.POINTER(abi.PrimitiveOmm), u32]
    L.b200pt_set_environment.argtypes = [vp, f32p, i32, i32, C.POINTER(C.c_float)]
    L.b200pt_resize.argtypes = [vp, i32, i32, i32, i32]
    L.b200pt_resize_interleaved.argtypes = [vp, i32, i32, i32, i32, i32]
    L.b200pt_read_accum_async.argtypes = [vp, vp, C.c_size_t, i32]
    L.b200pt_wait_read.argtypes = [vp, i32]
    L.b200pt_set_frames_in_flight.argtypes = [vp, i32]
    L.b200pt_render_frame.argtypes = [vp, C.POINTER(abi.FrameInfo), C.POINTER(abi.PushConstant)]
    L.b200pt_synchronize.argtypes = [vp]
    L.b200pt_get_accum_device.argtypes = [vp, C.POINTER(vp), C.POINTER(C.c_size_t)]
    L.b200pt_read_accum.argtypes = [vp, f32p, C.c_size_t]
    L.b200pt_set_accum_device.argtypes = [vp, vp, C.c_size_t]
    L.b200pt_stream.argtypes = [vp]
    L.b200pt_stream.restype = vp
    L.b200pt_get_stats.argtypes = [vp, C.POINTER(abi.Stats)]
    L.b200pt_reset_stats.argtypes = [vp]
    L.b200pt_set_profiling.argtypes = [vp, i32]
    L.b200pt_trace_closest.argtypes = [vp, vp, u32, vp, vp]
    L.b200pt_trace_shadow.argtypes = [vp, vp, u32, vp, vp]
    L.b200pt_bvh_info.argtypes = [vp, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(u32), C.POINTER(u32)]
    L.b200pt_bsdf_eval.argtypes = [vp, vp, u32, vp]
    L.b200pt_bsdf_sample.argtypes = [vp, vp, u32, vp]
    L.b200pt_texture_lookup.argtypes = [vp, vp, u32, vp]
    L.b200pt_shade_state.argtypes = [vp, vp, u32, vp, vp]
    L.b200pt_read_selection.argtypes = [vp, vp, vp, C.c_size_t]
    L.b200pt_set_frame_batch.argtypes = [vp, i32]
    L.b200pt_flush.argtypes = [vp]
    L.b200pt_set_bvh_builder.argtypes = [vp, i32]
    L.b200pt_bvh_build_ms.argtypes = [vp, C.POINTER(C.c_double)]
    L.b200pt_update_transforms.argtypes = [vp, C.POINTER(abi.RenderNode), u32]
    L.b200pt_set_animation.argtypes = [vp, C.POINTER(abi.MorphTask), u32, C.POINTER(abi.SkinTask), u32]
    L.b200pt_animate.argtypes = [vp, vp, vp, vp]
    L.b200pt_set_node_hierarchy.argtypes = [vp, C.POINTER(abi.NodeHierarchy)]
    L.b200pt_update_node_matrices.argtypes = [vp, vp]
    L.b200pt_update_materials.argtypes = [vp, C.POINTER(abi.ShadeMaterial), u32, C.POINTER(abi.TextureInfo), u32]
    L.b200pt_update_node_materials.argtypes = [vp, C.POINTER(C.c_int32), u32]
    L.b200pt_update_lights.argtypes = [vp, C.POINTER(abi.Light), u32]
    L.b200pt_set_node_visibility.argtypes = [vp, C.POINTER(C.c_uint8), u32]
    L.b200pt_tonemap.argtypes = [vp, C.POINTER(abi.Tonemapper), vp, C.c_size_t, C.POINTER(C.c_float)]
    L.b200pt_tonemap_image.argtypes = [vp, C.POINTER(abi.Tonemapper), vp, i32, i32, vp, C.POINTER(C.c_float)]
    L.b200pt_get_tonemapped_device.argtypes = [vp, C.POINTER(vp), C.POINTER(C.c_size_t)]
    L.b200pt_set_guide_outputs.argtypes = [vp, i32]
    L.b200pt_read_guide.argtypes = [vp, vp, C.c_size_t]
    L.b200pt_get_guide_device.argtypes = [vp, C.POINTER(vp), C.POINTER(C.c_size_t)]
    L.b200pt_set_dlss_guides.argtypes = [vp, i32]
    L.b200pt_read_dlss_guides.argtypes = [vp, C.POINTER(abi.DlssGuides)]
    L.b200pt_get_dlss_guides_device.argtypes = [vp, C.POINTER(abi.DlssGuides)]
    L.b200pt_get_selection_device.argtypes = [vp, C.POINTER(vp), C.POINTER(vp)]
    for name in EXPORTS:
        getattr(L, name)  # raises AttributeError if a declared symbol is not exported
    _libs[path] = L
    return L
