"""Packing of hit-state unit-test records for b200pt_shade_state (include/b200pt.h).

Input, 16 floats per record:
  0-2 ray origin | 3 tmin | 4-6 ray direction | 7 tmax  (the ray of b200pt_trace_closest) |
  8 isInside (0 / 1) | 9 coneWidth | 10 pixelAngle (cone spread per unit distance) | 11 texGradScale | 12-15 unused

Output, 96 floats per record: the closest hit, the HitState getHitState returns for it, the texture gradient of the
ray-cone footprint and the PbrMaterial evaluateMaterial returns.  A miss has t = 1e32, node = prim = tri = -1 and zeros
elsewhere.  Ids are stored as float values.
"""
import numpy as np

IN_FLOATS = 16
OUT_FLOATS = 96
MISS_T = np.float32(1e32)

# name -> (first float, width)
FIELDS = dict(
    t=(0, 1), node=(1, 1), prim=(2, 1), tri=(3, 1), u=(4, 1), v=(5, 1),
    # HitState (get_hit.h.slang:26-38)
    pos=(6, 3), nrm=(9, 3), color=(12, 4), geonrm=(16, 3), shadowPos=(19, 3), uv0=(22, 2), uv1=(24, 2),
    tangent=(26, 3), bitangent=(29, 3), texelDensity=(32, 1),
    # worldFoot * texelDensity * texGradScale (gltf_pathtrace.slang:164,196)
    texGrad=(33, 1),
    # PbrMaterial as evaluateMaterial leaves it (gltf_material_eval.h.slang:168-457)
    baseColor=(34, 3), opacity=(37, 1), roughness=(38, 2), metallic=(40, 1), emissive=(41, 3),
    N=(44, 3), T=(47, 3), B=(50, 3), Ng=(53, 3), ior1=(56, 1), ior2=(57, 1), specular=(58, 1), specularColor=(59, 3),
    transmission=(62, 1), attenuationColor=(63, 3), attenuationDistance=(66, 1), thickness=(67, 1),
    clearcoat=(68, 1), clearcoatRoughness=(69, 1), Nc=(70, 3), iridescence=(73, 1), iridescenceIor=(74, 1),
    iridescenceThickness=(75, 1), sheenColor=(76, 3), sheenRoughness=(79, 1), dispersion=(80, 1),
    diffuseTransmissionFactor=(81, 1), diffuseTransmissionColor=(82, 3), scatterCoefficient=(85, 3),
    scatterAnisotropy=(88, 1), retroreflection=(89, 1),
)
HIT_FIELDS = ("pos", "nrm", "color", "geonrm", "shadowPos", "uv0", "uv1", "tangent", "bitangent", "texelDensity")
MATERIAL_FIELDS = tuple(k for k in FIELDS if FIELDS[k][0] >= 34)


def records(rays, *, inside=0.0, cone_width=0.0, pixel_angle=0.0, tex_grad_scale=1.0):
    """One record per ray (float [n, 8] as b200pt_trace_closest takes them); the scalars broadcast."""
    rays = np.asarray(rays, np.float32).reshape(-1, 8)
    r = np.zeros((len(rays), IN_FLOATS), np.float32)
    r[:, 0:8] = rays
    r[:, 8] = inside
    r[:, 9] = cone_width
    r[:, 10] = pixel_angle
    r[:, 11] = tex_grad_scale
    return r


def field(out, name):
    """[n] or [n, width] view of one field of the output records"""
    a, w = FIELDS[name]
    out = np.asarray(out).reshape(-1, OUT_FLOATS)
    return out[:, a] if w == 1 else out[:, a:a + w]
