"""The CPU oracle's getHitState and evaluateMaterial (through Oracle.shade_state) against the float64 restatement of
tests/hitref.py, on the material zoo, its sampler variant and an attribute-and-transform zoo built here.

What is asserted, per record that hits:
  1. independent of any restatement, on the world-space vertices in float64: hit.pos = org + t dir; geonrm parallel to the
     world-space face normal and facing the ray; texelDensity = sqrt(uv area / world area); the shading N, T, B unit and
     T perpendicular to N;
  2. every field within TOL of hitref (below); a record within hitref.EPS of a branch threshold is accepted on either side
     of it, such records stay under 1 % and every branch is taken both ways somewhere.

Tolerances (fp32 implementation against float64; |x| is the reference value):
  * geometry (pos, shadowPos): 2e-6 * (1 + |coordinates|): a handful of fp32 roundings of an object-to-world affine map;
  * unit vectors, uv, colour, texel density, texGrad and untextured factors: 2e-5 absolute + 2e-5 relative: normalise,
    cross and the sqrt of the density each add a few ulp, and the texture gradient compounds about ten of them;
  * values fetched from textures and everything built on them (normal-mapped frames, anisotropic roughness): 5e-4 absolute:
    the fp32 uv of a hit differs from the float64 one by a few ulp of |uv| <= 8, which moves a linear fetch on a 64-texel
    level by up to 8 * 2^-21 * 64 texels times the largest step between neighbouring texels (< 1);
  * the tangent frame (tangent, bitangent and the material's N, T, B, Nc built on it): the above times 1 / |t - n (n.t)|
    for the unit object-space tangent t, since the projection against the normal cancels when t leans towards n;
  * texGrad: the above plus 4e-7 relative over max(|N.V|, 1e-3): the ray-cone footprint divides by that cosine, so the fp32
    error of the geometric normal grows as the hit grazes;
  * scatterCoefficient: relative 1e-4 (it goes through logf) plus 1e-6 of the attenuation coefficient: the single-scatter
    albedo 1 - t^2 cancels to a few ulp of 1 when the multi-scatter colour is small.
"""
import math

import numpy as np
import pytest

import hitref
from test_texture_sampling import check_chain, read_levels
from vk_gltf_renderer_b200 import shade_io, synth
from vk_gltf_renderer_b200.scene import Camera, Scene

GEOMETRY = ("pos", "shadowPos")
FRAME = ("tangent", "bitangent", "N", "T", "B", "Nc")
TEXTURED = ("baseColor", "opacity", "roughness", "metallic", "emissive", "N", "T", "B", "Nc", "specular", "specularColor",
            "thickness", "transmission", "clearcoat", "clearcoatRoughness", "iridescence", "iridescenceThickness",
            "sheenColor", "sheenRoughness", "diffuseTransmissionFactor", "diffuseTransmissionColor", "ior1", "ior2")


# ---- scenes ------------------------------------------------------------------------------------------------------------
def _noise(rng, size, lo=0.0, hi=1.0):
    return synth._u8(lo + (hi - lo) * synth.value_noise(size, 4, rng, 4))


def _pack(rgba):
    c = synth._u8(np.asarray(rgba)).astype(np.uint32)
    return c[:, 0] | (c[:, 1] << 8) | (c[:, 2] << 16) | (c[:, 3] << 24)


def attribute_zoo(seed=7):
    """Primitives with each useful subset of {normals, uv0, uv1, colours, tangents}, under non-uniform scale, shear and a
    mirror, a double-sided open sheet, vertex normals against the face, a coarse sphere, a zero-uv-area triangle, and the
    material edges of hitref's branches (see the module docstring of test_shade_state)."""
    rng = np.random.default_rng(seed)
    scn = Scene()
    t_rgb = scn.add_texture(_noise(rng, 32), srgb=True)
    t_lin = scn.add_texture(_noise(rng, 23, 0.2, 0.9), wrapS=33648, wrapT=33071)
    t_nm = scn.add_texture(synth.make_texture_set(32, rng, (0.8, 0.8, 0.8))[2])
    t_near = scn.add_texture(_noise(rng, 16), magFilter=9728, minFilter=9984)
    t_sg = scn.add_texture(synth._u8(np.concatenate([np.broadcast_to(np.linspace(0.0, 0.15, 32)[None, :, None], (32, 32, 3)),
                                                     np.full((32, 32, 1), 0.7)], -1)))
    c, s = math.cos(0.7), math.sin(0.7)
    rot = (1.6 * c, 1.6 * s, -0.9 * s, 0.9 * c, 0.3, -0.2)        # rotated, scaled KHR_texture_transform
    ti = scn.add_texture_info
    mats = [
        # 0: TEXCOORD_1 base colour under a rotated transform, a normal map scaled by -0.7, a clearcoat normal
        scn.add_material(pbrBaseColorFactor=[0.9, 0.8, 0.7, 1], pbrRoughnessFactor=0.5, pbrMetallicFactor=0.0, pbrBaseColorTexture=ti(t_rgb, 1, rot),
                         normalTexture=ti(t_nm), normalTextureScale=-0.7, clearcoatFactor=0.8, clearcoatNormalTexture=ti(t_nm, 1, rot)),
        # 1: a normal map scaled by 2.5, metallic-roughness fetched NEAREST, double-sided
        scn.add_material(pbrBaseColorFactor=[0.5, 0.6, 0.7, 1], pbrRoughnessFactor=0.8, pbrMetallicFactor=0.7, normalTexture=ti(t_nm, 0, rot),
                         normalTextureScale=2.5, pbrMetallicRoughnessTexture=ti(t_near), doubleSided=1),
        # 2: anisotropy with a direction texture, iridescence with thickness maximum 0
        scn.add_material(pbrBaseColorFactor=[0.8, 0.6, 0.3, 1], pbrRoughnessFactor=0.4, pbrMetallicFactor=1.0, anisotropyStrength=0.7,
                         anisotropyRotation=[math.sin(-1.1), math.cos(-1.1)], anisotropyTexture=ti(t_lin, 1), iridescenceFactor=1.0,
                         iridescenceThicknessMinimum=100.0, iridescenceThicknessMaximum=0.0),
        # 3: anisotropy without a texture, iridescence with a thickness texture
        scn.add_material(pbrBaseColorFactor=[0.3, 0.6, 0.8, 1], pbrRoughnessFactor=0.3, pbrMetallicFactor=0.0, anisotropyStrength=0.5,
                         anisotropyRotation=[math.sin(0.4), math.cos(0.4)], iridescenceFactor=0.8, iridescenceThicknessMinimum=-50.0,
                         iridescenceThicknessMaximum=400.0, iridescenceThicknessTexture=ti(t_lin)),
        # 4: spec-gloss, specular below, inside and above the smoothstep ramp across the texture
        scn.add_material(pbrModel=1, pbrDiffuseFactor=[0.7, 0.6, 0.5, 1], pbrSpecularFactor=[1.0, 0.8, 0.9], pbrGlossinessFactor=0.9,
                         pbrSpecularGlossinessTexture=ti(t_sg), pbrDiffuseTexture=ti(t_rgb)),
        # 5: spec-gloss by factors alone: inside the ramp
        scn.add_material(pbrModel=1, pbrDiffuseFactor=[0.9, 0.9, 0.9, 1], pbrSpecularFactor=[0.07, 0.06, 0.02], pbrGlossinessFactor=0.5),
        # 6: negative emissive factor
        scn.add_material(pbrBaseColorFactor=[0.4, 0.4, 0.4, 1], emissiveFactor=[-1.0, 0.5, 2.0], emissiveTexture=ti(t_rgb)),
        # 7: scattering medium with attenuation colour 0 and distance 0, thickness 0
        scn.add_material(pbrBaseColorFactor=[1, 1, 1, 1], transmissionFactor=1.0, attenuationColor=[0.0, 0.5, 0.0], attenuationDistance=0.0,
                         multiscatterColorFactor=[0.5, 0.3, 0.0], scatterAnisotropy=0.3, thicknessFactor=0.0),
        # 8: volume with thickness > 0 and a thickness texture, transmission texture
        scn.add_material(pbrBaseColorFactor=[0.9, 0.95, 1, 1], transmissionFactor=0.9, transmissionTexture=ti(t_lin), ior=1.33,
                         thicknessFactor=0.6, thicknessTexture=ti(t_lin, 1), attenuationColor=[0.6, 0.7, 0.8], attenuationDistance=2.0,
                         doubleSided=1),
    ]
    quad_p = np.array([[-0.5, -0.5, 0], [0.5, -0.5, 0], [0.5, 0.5, 0], [-0.5, 0.5, 0]], np.float32)
    quad_i = np.array([[0, 1, 2], [0, 2, 3]], np.uint32)
    uv = np.array([[0, 0], [2, 0], [2, 2], [0, 2]], np.float32)
    tilt = np.array([[0.3, 0.1, 1], [-0.2, 0.4, 1], [0.1, -0.3, 1], [0.0, 0.2, 1]], np.float32)
    tilt /= np.linalg.norm(tilt, axis=1, keepdims=True)
    col = _pack([[1, 0.5, 0.2, 0.3], [0.2, 1, 0.4, 1.0], [0.6, 0.3, 1, 0.6], [0.9, 0.9, 0.1, 0.8]])
    tan = np.array([[1, 0, 0, 1], [1, 0.1, 0, -1], [0.9, 0.2, 0.1, 1], [1, -0.1, 0, -1]], np.float32)
    prims = [
        scn.add_primitive(quad_p, quad_i, normals=tilt),                                                  # 0 normals only
        scn.add_primitive(quad_p, quad_i, uv1=uv * 0.7 + 0.1, colors=col),                                 # 1 uv1 without uv0, colours
        scn.add_primitive(quad_p, quad_i, normals=tilt, uv0=uv, uv1=uv[::-1] * 1.3, colors=col, tangents=tan),  # 2 everything, w varies
        scn.add_primitive(quad_p * [1, 1, 1], quad_i[:, ::-1].copy()),                                    # 3 nothing, facing -z
        scn.add_primitive(quad_p, quad_i, normals=-tilt, uv0=uv),                                          # 4 normals against the face
        scn.add_primitive(np.array([[-0.5, -0.5, 0], [0.5, -0.5, 0], [0, 0.5, 0]], np.float32), np.array([[0, 1, 2]], np.uint32),
                          uv0=np.array([[0.3, 0.3]] * 3, np.float32), uv1=np.array([[0, 0], [1, 0], [0, 1]], np.float32)),  # 5 zero uv area
        scn.add_primitive(quad_p, quad_i, normals=tilt, uv0=uv, uv1=uv * 0.5, tangents=tan),               # 6 no colours
    ]
    sp = synth._sphere(0.0, 0.0, 0.0, 0.5, n=6)
    prims.append(scn.add_primitive(sp[0], sp[4], normals=sp[1], uv0=sp[2], uv1=sp[2] * 2.0))               # 7 coarse sphere, no tangents

    def xf(tx, ty, tz, lin=np.eye(3)):
        m = np.eye(4)
        m[:3, :3] = lin
        m[:3, 3] = [tx, ty, tz]
        return m
    shear = np.array([[1.4, 0.5, 0.0], [0.0, 0.6, 0.3], [0.2, 0.0, 1.1]])
    mirror = np.diag([-1.0, 1.0, 1.0]) @ np.array([[0.9, 0.0, 0.2], [0.1, 1.2, 0.0], [0.0, 0.0, 0.8]])
    place = [
        (0, 0, xf(-3, 0, 0)), (1, 1, xf(-2, 0, 0, shear)), (2, 0, xf(-1, 0, 0)), (3, 3, xf(0, 0, 0)), (4, 1, xf(1, 0, 0)),
        (5, 6, xf(2, 0, 0)), (6, 2, xf(3, 0, 0, shear)), (7, 4, xf(-3, 1.5, 0)), (7, 5, xf(-2, 1.5, 0, mirror)), (2, 8, xf(-1, 1.5, 0, mirror)),
        (7, 7, xf(0, 1.5, 0)), (6, 8, xf(1, 1.5, 0, shear)), (7, 3, xf(2, 1.5, 0, shear)), (0, 2, xf(3, 1.5, 0, mirror)),
        (6, 1, xf(-2, -1.5, 0, mirror @ shear)), (1, 8, xf(0, -1.5, 0)), (4, 0, xf(2, -1.5, 0, mirror)),
    ]
    for p, m, M in place:
        scn.add_node(prims[p], mats[m], M)
    cam = Camera()
    cam.eye = np.array([0.0, 0.0, 6.0], np.float32)
    scn.camera = cam
    return scn


def add_readback(scene):
    """one identity texture info per texture, for read_levels; returns the image dicts test_texture_sampling uses"""
    ims = []
    for k, t in enumerate(scene.textures):
        h, w = t["rgba8"].shape[:2]
        ims.append(dict(w=w, h=h, srgb=bool(t["srgb"]), rgba8=t["rgba8"], readback=scene.add_texture_info(k)))
    return ims


def stored_levels(lookup, ims):
    """every texture's levels, read back through the implementation's lookup and checked against the float64 blit"""
    levels = {}
    for k, im in enumerate(ims):
        lv, beyond = read_levels(lookup, None, im)
        check_chain(lv, beyond, im)
        levels[k] = lv
    return levels


def aimed_rays(scene, n_per_node, seed, prims=None, nodes=None, both_sides=True):
    """rays at random interior points of random triangles of every visible node, from either side, some at grazing
    angles; plus rays that miss"""
    rng = np.random.default_rng(seed)
    prims = scene.render_prims if prims is None else prims
    nodes = scene.render_nodes if nodes is None else nodes
    out = []
    for rn in nodes:
        if not rn.get("visible", True):
            continue
        P = prims[rn["renderPrimID"]]
        M = np.asarray(rn["objectToWorld"], np.float64).reshape(4, 4).T
        pv = np.asarray(P["positions"], np.float64)[np.asarray(P["indices"], np.int64)]
        good = np.flatnonzero(np.linalg.norm(np.cross(pv[:, 1] - pv[:, 0], pv[:, 2] - pv[:, 0]), axis=1) > 1e-12)  # not the poles' slivers
        tri = good[rng.integers(0, len(good), n_per_node)]
        b = rng.dirichlet((1.0, 1.0, 1.0), n_per_node)
        v = np.asarray(P["positions"], np.float64)[np.asarray(P["indices"], np.int64)[tri]]
        obj = np.einsum("nk,nkj->nj", b, v)
        target = obj @ M[:3, :3].T + M[:3, 3]
        fn = np.cross(v[:, 1] - v[:, 0], v[:, 2] - v[:, 0]) @ np.linalg.inv(M[:3, :3])
        fn /= np.linalg.norm(fn, axis=1, keepdims=True)
        d = rng.normal(size=(n_per_node, 3))
        d /= np.linalg.norm(d, axis=1, keepdims=True)
        side = np.where(rng.random(n_per_node) < (0.3 if both_sides else 0.0), 1.0, -1.0)
        d = np.where((np.sum(d * fn, 1) * side)[:, None] < 0, -d, d)
        graze = rng.random(n_per_node) < 0.15
        d[graze] = d[graze] - fn[graze] * np.sum(d[graze] * fn[graze], 1)[:, None] * 0.97
        d /= np.linalg.norm(d, axis=1, keepdims=True)
        dist = rng.uniform(0.2, 3.0, n_per_node)
        org = target - d * dist[:, None]
        out.append(np.concatenate([org, np.full((n_per_node, 1), 1e-4), d, np.full((n_per_node, 1), 1e30)], 1))
    miss = np.tile(np.array([[0, 50, 0, 0, 0, 1, 0, 1e30]]), (4, 1))
    out.append(miss)
    return np.concatenate(out).astype(np.float32)


def sweep_records(rays, seed, cone=(0.0, 0.0), scale=1.0):
    """isInside both ways and a ray-cone footprint that puts lambda on magnification, fractional levels, the nearest-mip
    rounding points and beyond the chain"""
    rng = np.random.default_rng(seed)
    r = shade_io.records(rays, inside=(rng.random(len(rays)) < 0.4).astype(np.float32))
    r[:, 9] = np.float32(cone[0]) * (2.0 ** rng.uniform(-6, 6, len(r))).astype(np.float32)
    r[:, 10] = np.float32(cone[1]) * (2.0 ** rng.uniform(-6, 6, len(r))).astype(np.float32)
    r[:, 11] = scale
    r[::7, 9:11] = 0.0
    return r


# ---- checks ------------------------------------------------------------------------------------------------------------
def world_triangles(scene, node, tri, prims=None, nodes=None):
    prims = scene.render_prims if prims is None else prims
    nodes = scene.render_nodes if nodes is None else nodes
    v = np.empty((len(node), 3, 3))
    uv = np.full((len(node), 3, 2), np.nan)
    for k, (nd, t) in enumerate(zip(node, tri)):
        rn = nodes[nd]
        P = prims[rn["renderPrimID"]]
        M = np.asarray(rn["objectToWorld"], np.float64).reshape(4, 4).T
        idx = np.asarray(P["indices"], np.int64)[t]
        v[k] = np.asarray(P["positions"], np.float64)[idx] @ M[:3, :3].T + M[:3, 3]
        if P["uv0"] is not None:
            uv[k] = np.asarray(P["uv0"], np.float64)[idx]
    return v, uv


def check_independent(scene, rec_in, out, tag, prims=None, nodes=None):
    """assertion group 1 (module docstring); returns the hit mask"""
    F = lambda name: shade_io.field(out, name).astype(np.float64)
    hit = F("t") < shade_io.MISS_T
    assert (F("node")[~hit] == -1).all() and (out[~hit, 4:] == 0).all(), tag
    o, d = rec_in[hit, 0:3].astype(np.float64), rec_in[hit, 4:7].astype(np.float64)
    node, tri = F("node")[hit].astype(np.int64), F("tri")[hit].astype(np.int64)
    v, uv = world_triangles(scene, node, tri, prims, nodes)
    # t of a grazing hit carries the fp32 error of the intersection divided by the cosine
    cos = np.maximum(np.abs(np.sum(F("geonrm")[hit] * d, 1)), 1e-2)
    scale = (1.0 + np.abs(o).max(1) + F("t")[hit]) / cos
    err = np.linalg.norm(F("pos")[hit] - (o + F("t")[hit, None] * d), axis=1)
    assert (err < 2e-6 * scale).all(), (tag, "pos != org + t dir", err.max(), np.flatnonzero(err >= 2e-6 * scale)[:5])
    fn = np.cross(v[:, 1] - v[:, 0], v[:, 2] - v[:, 0])
    area = np.linalg.norm(fn, axis=1)
    fn /= area[:, None]
    g = F("geonrm")[hit]
    assert (np.linalg.norm(np.cross(g, fn), axis=1) < 1e-4).all(), (tag, "geonrm not parallel to the face")
    assert (np.sum(g * d, 1) <= 1e-6).all(), (tag, "geonrm does not face the ray")
    has_uv = np.isfinite(uv[:, 0, 0])
    duv1, duv2 = uv[:, 1] - uv[:, 0], uv[:, 2] - uv[:, 0]
    dens = np.sqrt(np.maximum(np.abs(duv1[:, 0] * duv2[:, 1] - duv1[:, 1] * duv2[:, 0]), 1e-20) / np.maximum(area, 1e-20))
    td = F("texelDensity")[hit]
    assert np.allclose(td[has_uv], dens[has_uv], rtol=1e-4, atol=1e-9), (tag, "texelDensity")
    assert (td[~has_uv] == 0).all()
    for name in ("nrm", "tangent", "bitangent", "N", "T", "B"):
        assert (np.abs(np.linalg.norm(F(name)[hit], axis=1) - 1) < 1e-5).all(), (tag, name, "not unit")
    # T is orthogonal to N except where the reflect check replaced the shading normal by the geometric one
    replaced = np.all(out[hit, 9:12] == out[hit, 16:19], axis=1)
    dots = np.abs(np.sum(F("T")[hit] * F("N")[hit], 1))
    assert (dots[~replaced] < 1e-5).all(), (tag, "T not orthogonal to N", dots[~replaced].max())
    return hit


def tolerance(name, ref):
    ref = np.abs(ref)
    if name == "scatterCoefficient":
        return 1e-4 * ref + 1e-6
    if name in GEOMETRY:
        return 2e-6 * (1 + ref.max(-1, keepdims=True) if ref.ndim > 1 else 1 + ref)
    if name in TEXTURED:
        return 5e-4 + 2e-5 * ref
    return 2e-5 + 2e-5 * ref


def compare_reference(sref, rec_in, out, tag, fields=None, stats=None):
    """assertion group 2: every field against hitref, either side of a branch for the records near one"""
    hit = shade_io.field(out, "t") < shade_io.MISS_T
    F = lambda name: shade_io.field(out[hit], name).astype(np.float64)
    hits = (F("node").astype(np.int64), F("tri").astype(np.int64), F("u"), F("v"), F("t"))
    ref, near, taken = sref.evaluate(rec_in[hit], hits)
    # the alternatives: each branch's near decisions taken the other way on their own, and all of a record's at once
    alts = [(near[b], sref.evaluate(rec_in[hit], hits, flip=near[b], only=b)[0]) for b in hitref.BRANCHES if near.get(b, np.zeros(1)).any()]
    if near["any"].any():
        alts.append((near["any"], sref.evaluate(rec_in[hit], hits, flip=near["any"])[0]))
    worst = {}
    for name in fields or [k for k in shade_io.FIELDS if shade_io.FIELDS[k][0] >= 6]:
        got = F(name)

        def excess(R):
            r = np.asarray(R[name], np.float64)
            tol = tolerance(name, r)
            if name in FRAME:
                tol = tol * sref.frame_cond[:, None]
            if name == "texGrad":
                # the footprint divides by |N.V|: the fp32 error of the geometric normal, relative to that cosine
                cos = np.maximum(np.abs(np.sum(R["geonrm"] * rec_in[hit, 4:7], 1)), 1e-3)
                tol = tol + 4e-7 * np.abs(r) / cos
            if name == "scatterCoefficient":
                # the single-scatter albedo is 1 - t^2 with t near 1 for a small albedo: a few ulp of 1, times the coefficient
                att = -np.log(np.maximum(R["attenuationColor"], 0.001)) / np.maximum(R["attenuationDistance"], 0.001)[:, None]
                tol = tol + 1e-6 * att
            e = np.abs(got - r) - tol
            return e.max(1) if e.ndim > 1 else e
        ok = excess(ref) <= 0
        for mask, R in alts:
            ok |= mask & (excess(R) <= 0)
        bad = np.flatnonzero(~ok)
        r = np.asarray(ref[name], np.float64)
        assert len(bad) == 0, (tag, name, len(bad), bad[:4], got[bad[:4]], r[bad[:4]])
        dev = np.abs(got - r)
        dev = dev.max(1) if dev.ndim > 1 else dev
        worst[name] = float(dev[~near["any"]].max()) if (~near["any"]).any() else 0.0
    n_near = int(near["any"].sum())
    assert n_near <= 0.01 * len(near["any"]), (tag, str({k: int(v.sum()) for k, v in near.items()}))
    if stats is not None:
        stats["records"] = stats.get("records", 0) + int(hit.sum())
        stats["near"] = stats.get("near", 0) + n_near
        for k, v in taken.items():
            stats.setdefault("taken", {}).setdefault(k, set()).update(v)
        for k, v in worst.items():
            stats.setdefault("worst", {})[k] = max(stats.get("worst", {}).get(k, 0.0), v)
    return ref, near


def run_scene(impl, scene, levels_of, rec_in, seeds, tag, stats, prims=None, nodes=None):
    """one implementation's records on one scene through both assertion groups; returns the records"""
    out = impl(rec_in, seeds.copy())
    hit = check_independent(scene, rec_in, out, tag, prims, nodes)
    assert hit.mean() > 0.5, (tag, hit.mean())
    sref = hitref.SceneRef(scene, levels_of, prims, nodes)
    compare_reference(sref, rec_in, out, tag, stats=stats)
    return out


def scenes():
    zoo = synth.synth_material_zoo()
    zoo_s = synth.synth_material_zoo(samplers=True)
    attr = attribute_zoo()
    return [("zoo", zoo, 64, (2e-3, 4e-3)), ("zoo_samplers", zoo_s, 64, (2e-3, 4e-3)), ("attributes", attr, 160, (4e-3, 8e-3))]


BRANCH_SIDES = ("frontFace", "sideFlip", "reflect", "fastTangent", "smoothstep", "iridescence", "iorSwap")


@pytest.fixture(scope="module")
def oracle_stats(oracle_mod):
    stats = {}
    for k, (tag, scn, per_node, cone) in enumerate(scenes()):
        ims = add_readback(scn)
        o = oracle_mod.Oracle()
        o.set_scene(scn)
        levels = stored_levels(o.texture_lookup, ims)
        rays = aimed_rays(scn, per_node, seed=100 + k)
        rec = sweep_records(rays, seed=200 + k, cone=cone)
        seeds = np.arange(len(rec), dtype=np.uint32) * 2654435761
        run_scene(lambda r, s: o.shade_state(r, s), scn, levels, rec, seeds, tag, stats)
    return stats


def test_oracle_hit_state_and_material_match_float64_reference(oracle_stats):
    s = oracle_stats
    print(f"oracle vs hitref: {s['records']} hits, {s['near']} within a branch margin")
    for k, v in sorted(s["worst"].items()):
        print(f"  {k:28s} {v:.3e}")
    for b in BRANCH_SIDES:
        assert s["taken"].get(b) == {False, True}, (b, s["taken"].get(b))
