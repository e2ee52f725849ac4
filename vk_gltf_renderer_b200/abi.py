"""ctypes mirror of include/b200pt.h (the C-ABI structs).

The POD structs are consumed by the CUDA library (libb200pt.so); the parity tests hand the very same bytes
to their CPU checker, so both sides see identical inputs.

Layouts follow the reference's host<->device structs:
  GltfRenderNode / GltfTextureInfo / GltfShadeMaterial / GltfLight  shaders/gltf_scene_io.h.slang:41-310
  SceneFrameInfo / PathtracePushConstant                           shaders/shaderio.h:148-196
"""
import ctypes as C

import numpy as np

c_float_p = C.POINTER(C.c_float)
c_u32_p = C.POINTER(C.c_uint32)
c_u8_p = C.POINTER(C.c_uint8)


class RenderNode(C.Structure):
    _fields_ = [("objectToWorld", C.c_float * 16), ("worldToObject", C.c_float * 16),
                ("materialID", C.c_int32), ("renderPrimID", C.c_int32)]


class RenderPrimitive(C.Structure):
    _fields_ = [("indices", c_u32_p), ("positions", c_float_p), ("normals", c_float_p),
                ("colors", c_u32_p), ("tangents", c_float_p), ("texCoords", c_float_p * 2),
                ("triangleCount", C.c_uint32), ("vertexCount", C.c_uint32)]


class TextureInfo(C.Structure):
    _fields_ = [("uvTransform", C.c_float * 6), ("index", C.c_int32), ("texCoord", C.c_int32)]


_MAT_FLOAT_FIELDS = [
    ("pbrBaseColorFactor", C.c_float * 4), ("emissiveFactor", C.c_float * 3), ("normalTextureScale", C.c_float),
    ("pbrRoughnessFactor", C.c_float), ("pbrMetallicFactor", C.c_float), ("alphaMode", C.c_int32),
    ("alphaCutoff", C.c_float), ("occlusionStrength", C.c_float), ("doubleSided", C.c_int32),
    ("attenuationColor", C.c_float * 3), ("ior", C.c_float), ("transmissionFactor", C.c_float),
    ("thicknessFactor", C.c_float), ("attenuationDistance", C.c_float), ("clearcoatFactor", C.c_float),
    ("specularColorFactor", C.c_float * 3), ("clearcoatRoughness", C.c_float), ("specularFactor", C.c_float),
    ("unlit", C.c_int32), ("iridescenceFactor", C.c_float), ("iridescenceThicknessMinimum", C.c_float),
    ("iridescenceThicknessMaximum", C.c_float), ("iridescenceIor", C.c_float),
    ("anisotropyRotation", C.c_float * 2), ("sheenColorFactor", C.c_float * 3), ("anisotropyStrength", C.c_float),
    ("sheenRoughnessFactor", C.c_float), ("dispersion", C.c_float), ("pbrModel", C.c_int32),
    ("pbrDiffuseFactor", C.c_float * 4), ("pbrSpecularFactor", C.c_float * 3), ("pbrGlossinessFactor", C.c_float),
    ("diffuseTransmissionColor", C.c_float * 3), ("diffuseTransmissionFactor", C.c_float),
    ("retroreflectionFactor", C.c_float), ("multiscatterColorFactor", C.c_float * 3), ("scatterAnisotropy", C.c_float),
]
MATERIAL_TEXTURE_SLOTS = [
    "pbrBaseColorTexture", "normalTexture", "pbrMetallicRoughnessTexture", "emissiveTexture", "occlusionTexture",
    "transmissionTexture", "thicknessTexture", "clearcoatTexture", "clearcoatRoughnessTexture",
    "clearcoatNormalTexture", "specularTexture", "specularColorTexture", "iridescenceTexture",
    "iridescenceThicknessTexture", "anisotropyTexture", "sheenColorTexture", "sheenRoughnessTexture",
    "pbrDiffuseTexture", "pbrSpecularGlossinessTexture", "diffuseTransmissionTexture",
    "diffuseTransmissionColorTexture", "retroreflectionTexture",
]


class ShadeMaterial(C.Structure):
    _fields_ = (_MAT_FLOAT_FIELDS + [(n, C.c_uint16) for n in MATERIAL_TEXTURE_SLOTS]
                + [("_pad16", C.c_uint16 * 2), ("_pad", C.c_uint64)])


class Light(C.Structure):
    _fields_ = [("direction", C.c_float * 3), ("type", C.c_int32), ("position", C.c_float * 3),
                ("radius", C.c_float), ("color", C.c_float * 3), ("intensity", C.c_float),
                ("angularSizeOrInvRange", C.c_float), ("innerAngle", C.c_float), ("outerAngle", C.c_float),
                ("_pad", C.c_int32)]


class Texture(C.Structure):
    _fields_ = [("rgba8", c_u8_p), ("width", C.c_int32), ("height", C.c_int32), ("srgb", C.c_int32),
                ("wrapS", C.c_int32), ("wrapT", C.c_int32), ("magFilter", C.c_int32), ("minFilter", C.c_int32)]


class SceneDesc(C.Structure):
    _fields_ = [("renderNodes", C.POINTER(RenderNode)), ("numRenderNodes", C.c_uint32),
                ("renderNodeVisible", c_u8_p),
                ("renderPrimitives", C.POINTER(RenderPrimitive)), ("numRenderPrimitives", C.c_uint32),
                ("materials", C.POINTER(ShadeMaterial)), ("numMaterials", C.c_uint32),
                ("textureInfos", C.POINTER(TextureInfo)), ("numTextureInfos", C.c_uint32),
                ("textures", C.POINTER(Texture)), ("numTextures", C.c_uint32),
                ("lights", C.POINTER(Light)), ("numLights", C.c_uint32)]


class FrameInfo(C.Structure):
    _fields_ = [("viewMatrix", C.c_float * 16), ("projInv", C.c_float * 16), ("viewInv", C.c_float * 16),
                ("viewProjMatrix", C.c_float * 16), ("prevMVP", C.c_float * 16), ("jitter", C.c_float * 2),
                ("imageSize", C.c_float * 2), ("flags", C.c_int32), ("envRotation", C.c_float),
                ("envBlur", C.c_float), ("envIntensity", C.c_float), ("backgroundColor", C.c_float * 3),
                ("visualization", C.c_int32), ("infinitePlaneDistance", C.c_float),
                ("infinitePlaneBaseColor", C.c_float * 3), ("infinitePlaneMetallic", C.c_float),
                ("infinitePlaneRoughness", C.c_float), ("shadowCatcherDarkenAmount", C.c_float)]


class PushConstant(C.Structure):
    _fields_ = [("maxDepth", C.c_int32), ("frameCount", C.c_int32), ("fireflyClampThreshold", C.c_float),
                ("texGradScale", C.c_float), ("numSamples", C.c_int32), ("totalSamples", C.c_int32),
                ("focalDistance", C.c_float), ("aperture", C.c_float), ("flags", C.c_int32),
                ("pixelAngle", C.c_float), ("mouseCoord", C.c_float * 2)]


class Stats(C.Structure):
    _fields_ = [("closestRays", C.c_uint64), ("shadowRays", C.c_uint64), ("shadedHits", C.c_uint64),
                ("pathsStarted", C.c_uint64), ("nodesVisited", C.c_uint64), ("trisTested", C.c_uint64),
                ("msTraceClosest", C.c_double), ("msTraceShadow", C.c_double), ("msShade", C.c_double),
                ("msOther", C.c_double), ("msTotal", C.c_double), ("kernelLaunches", C.c_uint64),
                ("launchesTraceClosest", C.c_uint64), ("launchesShade", C.c_uint64), ("launchesTraceShadow", C.c_uint64),
                ("msAnyHit", C.c_double), ("msResolve", C.c_double), ("launchesAnyHit", C.c_uint64), ("launchesResolve", C.c_uint64)]


class MicromapTriangle(C.Structure):
    """VkMicromapTriangleEXT (b200pt_micromap_triangle)"""
    _fields_ = [("dataOffset", C.c_uint32), ("subdivisionLevel", C.c_uint16), ("format", C.c_uint16)]


MICROMAP_TRIANGLE_DTYPE = np.dtype([("dataOffset", "<u4"), ("subdivisionLevel", "<u2"), ("format", "<u2")])


class Micromap(C.Structure):
    _fields_ = [("data", c_u8_p), ("dataSize", C.c_uint64), ("triangles", C.POINTER(MicromapTriangle)), ("numTriangles", C.c_uint32)]


class PrimitiveOmm(C.Structure):
    _fields_ = [("renderPrimID", C.c_uint32), ("micromap", C.c_uint32), ("baseTriangle", C.c_uint32),
                ("indices", C.POINTER(C.c_int32)), ("numIndices", C.c_uint32)]


class Tonemapper(C.Structure):
    """b200pt_tonemapper: the controls of nvshaders::TonemapperData the reference exposes (src/resources.hpp:212, its UI);
    method 0 filmic, 1 Uncharted 2, 2 clip, 3 ACES, 4 AgX, 5 Khronos PBR neutral"""
    _fields_ = [("method", C.c_int32), ("isActive", C.c_int32), ("exposure", C.c_float), ("brightness", C.c_float),
                ("contrast", C.c_float), ("saturation", C.c_float), ("vignette", C.c_float), ("autoExposure", C.c_int32)]


class DlssGuides(C.Structure):
    """b200pt_dlss_guides: the six DLSS guide planes (host or device pointers) and their sizes in bytes"""
    _fields_ = [("albedo", C.c_void_p), ("albedo_bytes", C.c_size_t), ("spec_albedo", C.c_void_p), ("spec_albedo_bytes", C.c_size_t),
                ("normal_roughness", C.c_void_p), ("normal_roughness_bytes", C.c_size_t), ("motion", C.c_void_p), ("motion_bytes", C.c_size_t),
                ("depth", C.c_void_p), ("depth_bytes", C.c_size_t), ("spec_hit_dist", C.c_void_p), ("spec_hit_dist_bytes", C.c_size_t)]


class Convergence(C.Structure):
    """b200pt_convergence: per-pixel stopping rule of an accumulation (include/b200pt.h); threshold 0 = off"""
    _fields_ = [("threshold", C.c_float), ("floor", C.c_float), ("minFrames", C.c_uint32), ("interval", C.c_uint32)]


class RenderNodeMapping(C.Structure):
    """b200pt_render_node_mapping == RenderNodeGpuMapping (shaders/world_matrix_io.h.slang:41-47)"""
    _fields_ = [("nodeID", C.c_int32), ("pad0", C.c_int32), ("materialID", C.c_int32), ("renderPrimID", C.c_int32)]


class NodeHierarchy(C.Structure):
    _fields_ = [("numNodes", C.c_uint32), ("numLevels", C.c_uint32), ("parentIndices", C.POINTER(C.c_int32)), ("topoNodeOrder", C.POINTER(C.c_int32)),
                ("levelOffsets", c_u32_p), ("mappings", C.POINTER(RenderNodeMapping)), ("instLocalMatrices", c_float_p)]


class MorphTask(C.Structure):
    """b200pt_morph_task (MorphPushConstant minus the per-frame / output pointers, shaders/animation_io.h.slang:45-59)"""
    _fields_ = [("renderPrimID", C.c_uint32), ("vertexCount", C.c_uint32), ("numTargets", C.c_uint32), ("_pad", C.c_uint32),
                ("basePositions", c_float_p), ("baseNormals", c_float_p), ("baseTangents", c_float_p),
                ("positionDeltas", c_float_p), ("normalDeltas", c_float_p), ("tangentDeltas", c_float_p)]


class SkinTask(C.Structure):
    """b200pt_skin_task (SkinPushConstant minus the per-frame / output pointers, shaders/animation_io.h.slang:29-43)"""
    _fields_ = [("renderPrimID", C.c_uint32), ("vertexCount", C.c_uint32), ("numJoints", C.c_uint32), ("_pad", C.c_uint32),
                ("basePositions", c_float_p), ("baseNormals", c_float_p), ("baseTangents", c_float_p),
                ("weights", c_float_p), ("joints", C.POINTER(C.c_int32))]


assert C.sizeof(MorphTask) == 64 and C.sizeof(SkinTask) == 56 and C.sizeof(Tonemapper) == 32

OMM_FORMAT_2_STATE, OMM_FORMAT_4_STATE = 1, 2
OMM_INDEX_FULLY_TRANSPARENT, OMM_INDEX_FULLY_OPAQUE, OMM_INDEX_FULLY_UNKNOWN_TRANSPARENT, OMM_INDEX_FULLY_UNKNOWN_OPAQUE = -1, -2, -3, -4
assert C.sizeof(MicromapTriangle) == 8

# sizes fixed by the reference's layouts (SURVEY.md §8a)
assert C.sizeof(RenderNode) == 136
assert C.sizeof(TextureInfo) == 32
assert C.sizeof(ShadeMaterial) == 288, C.sizeof(ShadeMaterial)
assert C.sizeof(Light) == 64
assert C.sizeof(FrameInfo) == 396
assert C.sizeof(PushConstant) == 48
assert ShadeMaterial.pbrRoughnessFactor.offset == 32 and ShadeMaterial.alphaMode.offset == 40
assert ShadeMaterial.occlusionStrength.offset == 48 and ShadeMaterial.doubleSided.offset == 52

SCENE_IS_ORTHOGRAPHIC = 1 << 0
SCENE_USE_SOLID_BACKGROUND = 1 << 1
SCENE_USE_HDR_ENVIRONMENT = 1 << 2
SCENE_USE_INFINITE_PLANE = 1 << 3
SCENE_INFINITE_PLANE_SHADOW_CATCHER = 1 << 4
PT_USE_DLSS = 1 << 0
PT_USE_OPTIX_DENOISER = 1 << 1
PT_FIRST_FRAME = 1 << 2

# b200pt_set_views / b200pt_render_views: the most views one handle renders at once, and the FrameInfo fields in which the views
# of one call may differ (every other byte must be equal)
MAX_VIEWS = 64
VIEW_POSE_FIELDS = ("viewMatrix", "viewInv", "viewProjMatrix", "prevMVP")


def fptr(a):
    """numpy float32 array -> float* (None -> NULL)."""
    if a is None:
        return c_float_p()
    assert a.dtype == np.float32 and a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(c_float_p)


def u32ptr(a):
    if a is None:
        return c_u32_p()
    assert a.dtype == np.uint32 and a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(c_u32_p)


def u8ptr(a):
    if a is None:
        return c_u8_p()
    assert a.dtype == np.uint8 and a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(c_u8_p)
