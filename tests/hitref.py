"""Float64 restatement of getHitState and evaluateMaterial, for the hit-state tests.

Restated statement by statement from the reference tree, in its default compile (every GLTF_USE_* = 1, USE_TEXTURES,
GLTF_USE_TEXTURE_TRANSFORM), reading the scene description (vk_gltf_renderer_b200.scene.Scene) and nothing of either
implementation:
  getHitState                    shaders/get_hit.h.slang:59-173
  computeTexelDensity            shaders/get_hit.h.slang:44-55
  vertex accessors               shaders/gltf_vertex_access.h.slang:81-133
  getTexture                     shaders/gltf_material_eval.h.slang:76-110
  convertSGToMR                  shaders/gltf_material_eval.h.slang:136-161
  multiToSingleScatterAlbedo     shaders/gltf_material_eval.h.slang:124-128
  evaluateMaterial               shaders/gltf_material_eval.h.slang:168-457
  texGrad = worldFoot * texelDensity * texGradScale      shaders/gltf_pathtrace.slang:164,196

The reference is followed where it looks odd: makeFastTangent of the unnormalised interpolated object-space normal
(get_hit.h.slang:139), the bitangent sign from tng[0].w only (:147), mul(worldToObject, n) for normals (:80,94), the
clearcoat normal built from pbrMat.T / B before the tangent update (gltf_material_eval.h.slang:341).

Three helpers are nvshaders code outside the reference tree, restated from their publications and UNPINNED:
  pointOffset            Hanika 2021, "Hacking the shadow terminator" (Ray Tracing Gems II, ch. 4): p + sum_i b_i t_i with
                         t_i = (p - p_i) - n_i min(0, (p - p_i).n_i)
  makeFastTangent        Frisvad 2012 ("Building an orthonormal basis from a 3D unit vector without normalization"):
                         tangent (1 - x^2/(1+z), -xy/(1+z), -x), w = 1, and (0, -1, 0) when z < -0.99998796
  rayConeWorldFootprint  Akenine-Moeller et al. 2021 ("Improved shader and texture level of detail using ray cones"):
                         (width + spread t) / max(|N.V|, 1e-3)

Textures are fetched through texref.TexRef on the levels the implementation stores (read back by the caller).

Branches with a threshold report their float64 margin so a test can accept either side of it: `evaluate(..., flip=mask,
only=name)` takes the decisions of branch `name` (every branch when None) that lie within its EPS of the threshold the other
way for the records in `mask`.
"""
import numpy as np

import texref as tr

MICROFACET_MIN_ROUGHNESS = np.float32(0.0014142)
# margins below which fp32 may take the other side of a branch (see the test module for the error model)
EPS = dict(frontFace=1e-5, sideFlip=1e-5, reflect=1e-5, fastTangent=1e-6, smoothstep=1e-5, iridescence=1e-6,
           bitangentSign=1e-5, texel=1e-3, lod=2e-5)
BRANCHES = tuple(EPS)


def _dot(a, b):
    return np.sum(a * b, -1)


def _norm(a):
    return a / np.linalg.norm(a, axis=-1, keepdims=True)


def _mix(a, b, c, bary):
    return a * bary[:, 0:1] + b * bary[:, 1:2] + c * bary[:, 2:3]


def _glm(m16):
    """glm column-major float[16] -> float64 (row, col) matrices [n, 4, 4]"""
    return np.asarray(m16, np.float64).reshape(-1, 4, 4).transpose(0, 2, 1)


def _unpack(c):
    c = np.asarray(c, np.uint32)
    return np.stack([(c >> s) & 0xFF for s in (0, 8, 16, 24)], -1).astype(np.float64) / 255.0


def point_offset(p, pa, pb, pc, na, nb, nc, bary):
    """Hanika 2021 (unpinned)"""
    out = p.copy()
    for pi, ni, k in ((pa, na, 0), (pb, nb, 1), (pc, nc, 2)):
        t = p - pi
        t = t - ni * np.minimum(0.0, _dot(t, ni))[:, None]
        out = out + t * bary[:, k:k + 1]
    return out


def make_fast_tangent(n):
    """Frisvad 2012 with the nvshaders threshold (unpinned); returns (tangent xyzw, margin n.z + 0.99998796)"""
    margin = n[:, 2] + 0.99998796
    a = 1.0 / (1.0 + n[:, 2])
    with np.errstate(divide="ignore", invalid="ignore"):
        t = np.stack([1.0 - n[:, 0] * n[:, 0] * a, -n[:, 0] * n[:, 1] * a, -n[:, 0], np.ones(len(n))], -1)
    return t, margin


def _smoothstep(e0, e1, x):
    t = np.clip((x - e0) / (e1 - e0), 0.0, 1.0)
    return t * t * (3.0 - 2.0 * t)


class SceneRef:
    """The scene description in float64.  `levels` maps texture index -> its stored levels (uint8 [h, w, 4], level 0
    first); `prims` optionally replaces render_prims (a posed copy from oracle/animation.apply); `nodes` optionally
    replaces render_nodes (matrices after the node hierarchy ran)."""

    def __init__(self, scene, levels, prims=None, nodes=None):
        self.scene = scene
        self.prims = scene.render_prims if prims is None else prims
        self.nodes = scene.render_nodes if nodes is None else nodes
        self._only = None
        self.tex = {}
        for k, t in enumerate(scene.textures):
            self.tex[k] = tr.TexRef(levels[k], bool(t["srgb"]), t["wrapS"], t["wrapT"], t["magFilter"], t["minFilter"])

    # ---- decisions ------------------------------------------------------------------------------------------------------
    def _take(self, name, margin, cond, flip, near):
        """cond (bool [n]) as float64 decides it, taken the other way where flip and |margin| < EPS; records near the
        threshold are marked in near[name]"""
        close = np.abs(margin) < EPS[name]
        near[name] = near.get(name, np.zeros(len(cond), bool)) | close
        return cond ^ (close & self._flips(name, flip))

    def _flips(self, name, flip):
        """the records whose decisions of branch `name` are taken the other way"""
        return flip if self._only in (None, name) else np.zeros_like(flip)

    # ---- getHitState (get_hit.h.slang:59-173) ---------------------------------------------------------------------------
    def hit_state(self, node, tri, u, v, ray_dir, flip, near, taken):
        n = len(node)
        node = np.asarray(node, np.int64)
        tri = np.asarray(tri, np.int64)
        O2W = _glm([self.nodes[k]["objectToWorld"] for k in node])
        W2O = _glm([self.nodes[k]["worldToObject"] for k in node])
        prim = np.array([self.nodes[k]["renderPrimID"] for k in node], np.int64)
        u, v = np.asarray(u, np.float64), np.asarray(v, np.float64)
        bary = np.stack([1.0 - u - v, u, v], -1)
        d = np.asarray(ray_dir, np.float64)

        def gather(name, width, fill=None):
            out = np.zeros((n, 3, width))
            has = np.zeros(n, bool)
            for p in np.unique(prim):
                m = prim == p
                a = self.prims[p][name]
                if a is None:
                    continue
                idx = np.asarray(self.prims[p]["indices"], np.int64)[tri[m]]
                vals = np.asarray(a)[idx]
                out[m] = _unpack(vals) if name == "colors" else np.asarray(vals, np.float64).reshape(-1, 3, width)
                has[m] = True
            return out, has

        P, _ = gather("positions", 3)
        p0, p1, p2 = P[:, 0], P[:, 1], P[:, 2]
        position = _mix(p0, p1, p2, bary)
        xp = lambda M, x: np.einsum("nij,nj->ni", M[:, :3, :3], x) + M[:, :3, 3]
        xv = lambda M, x: np.einsum("nij,nj->ni", M[:, :3, :3], x)
        xn = lambda M, x: np.einsum("nji,nj->ni", M[:, :3, :3], x)    # mul(worldToObject, float4(n, 0)): the transpose
        H = {}
        H["pos"] = xp(O2W, position)
        geo = _norm(np.cross(p1 - p0, p2 - p0))
        geonrm = _norm(xn(W2O, geo))
        Nv, has_n = gather("normals", 3)
        n0 = np.where(has_n[:, None], Nv[:, 0], geo)
        n1 = np.where(has_n[:, None], Nv[:, 1], geo)
        n2 = np.where(has_n[:, None], Nv[:, 2], geo)
        normal = np.where(has_n[:, None], _mix(n0, n1, n2, bary), geo)
        nrm = _norm(xn(W2O, normal))
        dg = _dot(geonrm, d) / np.linalg.norm(d, axis=-1)
        front = self._take("frontFace", dg, dg < 0, flip, near)
        taken.setdefault("frontFace", set()).update(set(front.tolist()))
        side = np.where(front, 1.0, -1.0)[:, None]
        H["shadowPos"] = xp(O2W, point_offset(position, p0, p1, p2, n0 * side, n1 * side, n2 * side, bary))
        T0, has_uv0 = gather("uv0", 2)
        T1, has_uv1 = gather("uv1", 2)
        H["uv0"] = np.where(has_uv0[:, None], _mix(T0[:, 0], T0[:, 1], T0[:, 2], bary), 0.0)
        H["uv1"] = np.where(has_uv1[:, None], _mix(T1[:, 0], T1[:, 1], T1[:, 2], bary), 0.0)
        self.has_uv = (has_uv0, has_uv1)      # a missing set reads (0, 0) exactly on both sides: no texel edge to doubt
        # computeTexelDensity (:44-55)
        we1, we2 = xv(O2W, p1 - p0), xv(O2W, p2 - p0)
        w_area = np.linalg.norm(np.cross(we1, we2), axis=-1)
        duv1, duv2 = T0[:, 1] - T0[:, 0], T0[:, 2] - T0[:, 0]
        uv_area = np.abs(duv1[:, 0] * duv2[:, 1] - duv1[:, 1] * duv2[:, 0])
        H["texelDensity"] = np.where(has_uv0, np.sqrt(np.maximum(uv_area, 1e-20) / np.maximum(w_area, 1e-20)), 0.0)
        C, has_c = gather("colors", 4)
        H["color"] = np.where(has_c[:, None], _mix(C[:, 0], C[:, 1], C[:, 2], bary), 1.0)
        Tg, has_t = gather("tangents", 4)
        ft, ft_margin = make_fast_tangent(normal)
        ft_margin = np.where(has_t, np.inf, ft_margin)
        below = self._take("fastTangent", ft_margin, ft_margin < 0, flip, near)
        taken.setdefault("fastTangent", set()).update(set(below[~has_t].tolist()))
        ft = np.where(below[:, None], np.array([0.0, -1.0, 0.0, 1.0]), ft)
        tng = np.where(has_t[:, None, None], Tg, ft[:, None, :])
        tangent = _norm(_mix(tng[:, 0, :3], tng[:, 1, :3], tng[:, 2, :3], bary))
        tangent = xv(O2W, tangent)
        resid = tangent - nrm * _dot(nrm, tangent)[:, None]
        # fp32 rounding of the projection is amplified by 1 / |residual| when the tangent leans towards the normal
        self.frame_cond = np.linalg.norm(tangent, axis=-1) / np.linalg.norm(resid, axis=-1)
        tangent = _norm(resid)
        bitangent = np.cross(nrm, tangent) * tng[:, 0, 3:4]
        geonrm = geonrm * side
        m = _dot(geonrm, nrm)
        fl = self._take("sideFlip", m, m < 0, flip, near)
        taken.setdefault("sideFlip", set()).update(set(fl.tolist()))
        s = np.where(fl, -1.0, 1.0)[:, None]
        nrm, tangent, bitangent = nrm * s, tangent * s, bitangent * s
        dn = _norm(d)
        r = dn - nrm * (2.0 * _dot(nrm, dn))[:, None]
        m = _dot(r, geonrm)
        rf = self._take("reflect", m, m < 0, flip, near)
        taken.setdefault("reflect", set()).update(set(rf.tolist()))
        nrm = np.where(rf[:, None], geonrm, nrm)
        H.update(nrm=nrm, geonrm=geonrm, tangent=tangent, bitangent=bitangent)
        return H

    # ---- getTexture (gltf_material_eval.h.slang:76-110) -----------------------------------------------------------------
    def texture(self, slot, rows, H, tex_grad, flip, near):
        """rgba float64 [len(rows), 4] of texture-info `slot` for the records `rows`"""
        ti = self.scene.texture_infos[slot]
        tc = H["uv1"][rows] if ti.texCoord else H["uv0"][rows]
        m = np.array(list(ti.uvTransform), np.float64)
        tt = np.stack([m[0] * tc[:, 0] + m[2] * tc[:, 1] + m[4], m[1] * tc[:, 0] + m[3] * tc[:, 1] + m[5]], -1)
        if ti.index < 0 or ti.index >= len(self.scene.textures):
            return np.ones((len(rows), 4))
        R = self.tex[ti.index]
        g = tex_grad[rows]
        lam = np.where(g > 0, R.lod(np.stack([m[0] * g, m[1] * g], -1), np.stack([m[2] * g, m[3] * g], -1)), -np.inf)
        # lambda on a level / rounding boundary: either side
        on = R.lod_boundaries(lam, EPS["lod"]) & (g > 0)
        near_rows = np.zeros(len(near["any"]), bool)
        near_rows[rows] = on
        near["lod"] = near.get("lod", np.zeros(len(near_rows), bool)) | near_rows
        fl = self._flips("lod", flip)[rows] & on
        b = np.where(np.abs(lam - np.round(lam)) < EPS["lod"], np.round(lam), np.floor(lam) + 0.5)
        lam = np.where(fl, np.where(lam < b, b + 1e-9, b - 1e-9), lam)
        # a nearest fetch whose texel-space coordinate lies on a texel edge: either texel
        lvl, linear = self._level_and_filter(R, lam)
        uv = tt.copy()
        on_edge = np.zeros(len(rows), bool)
        for k in range(2):
            size = np.array([max(1, (R.w0 if k == 0 else R.h0) >> int(l)) for l in lvl], np.float64)
            x = tt[:, k] * size
            e = np.abs(x - np.round(x)) < EPS["texel"]
            e &= ~linear & self.has_uv[ti.texCoord][rows]
            on_edge |= e
            alt = np.where(x < np.round(x), np.round(x) + 0.25, np.round(x) - 0.25) / size
            uv[:, k] = np.where(e & self._flips("texel", flip)[rows], alt, uv[:, k])
        near_rows = np.zeros(len(near["any"]), bool)
        near_rows[rows] = on_edge
        near["texel"] = near.get("texel", np.zeros(len(near_rows), bool)) | near_rows
        return R.sample(uv, np.where(g > 0, lam, -1.0))

    @staticmethod
    def _level_and_filter(R, lam):
        """(level sampled, whether it is filtered linearly) per query, for the texel-edge check"""
        mag = ~(lam > 0)
        lamc = np.minimum(np.where(mag, 0.0, lam), R.max_level)
        if R.mip_linear:
            lvl = np.floor(lamc)
        else:
            lvl = np.clip(np.ceil(lamc + 0.5) - 1, 0, R.max_level)
        lvl = np.where(mag, 0, lvl).astype(np.int64)
        return lvl, np.where(mag, R.mag_linear, R.min_linear)

    # ---- evaluateMaterial (gltf_material_eval.h.slang:168-457) ----------------------------------------------------------
    def material(self, node, H, inside, tex_grad, flip, near, taken):
        n = len(node)
        mat_of = np.array([max(0, self.nodes[k]["materialID"]) for k in node], np.int64)
        out = {}
        f = lambda name, w=1: np.array([np.array(list(getattr(self.scene.materials[m], name)), np.float64).reshape(w) for m in mat_of]).reshape(n, w) if w > 1 \
            else np.array([float(getattr(self.scene.materials[m], name)) for m in mat_of], np.float64)
        slots = lambda name: np.array([int(getattr(self.scene.materials[m], name)) for m in mat_of], np.int64)

        def tex(name, default):
            """the rgba of texture slot `name` where it is present (isTexturePresent: slot > 0), `default` elsewhere"""
            s = slots(name)
            res = np.broadcast_to(np.asarray(default, np.float64), (n, 4)).copy()
            for sl in np.unique(s[s > 0]):
                rows = np.flatnonzero(s == sl)
                res[rows] = self.texture(int(sl), rows, H, tex_grad, flip, near)
            return res, s > 0

        one = np.ones(4)
        sg = slots("pbrModel") == 1
        # specular-glossiness (:176-197 + convertSGToMR :136-161)
        diffuse = f("pbrDiffuseFactor", 4) * H["color"]
        diffuse = diffuse * tex("pbrDiffuseTexture", one)[0]
        sgt = tex("pbrSpecularGlossinessTexture", one)[0]
        specular = f("pbrSpecularFactor", 3) * sgt[:, :3]
        gloss = f("pbrGlossinessFactor") * sgt[:, 3]
        spec_i = specular.max(1)
        metal_sg = _smoothstep(0.05, 0.09, spec_i)
        m = np.where(sg, spec_i - 0.05, np.inf)
        is_metal = self._take("smoothstep", m, spec_i > 0.05, flip, near)
        taken.setdefault("smoothstep", set()).update(set(is_metal[sg].tolist()))
        base_sg = np.where(is_metal[:, None], specular, np.clip(diffuse[:, :3] / (1.0 - 0.04 * (1.0 - metal_sg))[:, None], 0, 1))
        r = 1.0 - gloss
        # metallic-roughness (:201-222)
        bc = f("pbrBaseColorFactor", 4) * H["color"] * tex("pbrBaseColorTexture", one)[0]
        mr = tex("pbrMetallicRoughnessTexture", one)[0]
        rough = np.maximum(f("pbrRoughnessFactor") * mr[:, 1], MICROFACET_MIN_ROUGHNESS)
        out["baseColor"] = np.where(sg[:, None], base_sg, bc[:, :3])
        out["opacity"] = np.where(sg, diffuse[:, 3], bc[:, 3])
        ra = np.where(sg, r * r, rough * rough)
        roughness = np.stack([ra, ra], -1)
        out["metallic"] = np.where(sg, metal_sg, np.clip(f("pbrMetallicFactor") * mr[:, 2], 0, 1))
        # normal map (:232-246): mul(normal_vector, float3x3(T, B, N))
        N, T, B, Ng = H["nrm"], H["tangent"], H["bitangent"], H["geonrm"]
        nt, has_nt = tex("normalTexture", one)
        nv = nt[:, :3] * 2.0 - 1.0
        nv = nv * np.stack([f("normalTextureScale"), f("normalTextureScale"), np.ones(n)], -1)
        pN = np.where(has_nt[:, None], _norm(T * nv[:, 0:1] + B * nv[:, 1:2] + N * nv[:, 2:3]), N)
        update = has_nt.copy()
        # emission (:249-254)
        out["emissive"] = np.maximum(0.0, f("emissiveFactor", 3) * tex("emissiveTexture", one)[0][:, :3])
        # volume (:256-269)
        out["attenuationColor"] = f("attenuationColor", 3)
        out["attenuationDistance"] = f("attenuationDistance")
        out["thickness"] = f("thicknessFactor") * tex("thicknessTexture", one)[0][:, 1]
        # specular (:271-285)
        out["specularColor"] = f("specularColorFactor", 3) * tex("specularColorTexture", one)[0][:, :3]
        out["specular"] = f("specularFactor") * tex("specularTexture", one)[0][:, 3]
        # ior swap inside a volume (:290-302)
        swap = np.asarray(inside, bool) & (out["thickness"] > 0)
        taken.setdefault("iorSwap", set()).update(set(swap.tolist()))
        out["ior1"] = np.where(swap, f("ior"), 1.0)
        out["ior2"] = np.where(swap, 1.0, f("ior"))
        # transmission (:304-311)
        out["transmission"] = f("transmissionFactor") * tex("transmissionTexture", one)[0][:, 0]
        # volume scatter (:313-323)
        ms = f("multiscatterColorFactor", 3)
        t = 4.09712 + 4.20863 * ms - np.sqrt(9.59217 + 41.6808 * ms + 17.7126 * ms * ms)
        ssa = 1.0 - t * t
        att = -np.log(np.maximum(out["attenuationColor"], 0.001)) / np.maximum(out["attenuationDistance"], 0.001)[:, None]
        out["scatterCoefficient"] = np.where((ms > 0).any(1)[:, None], att * ssa, 0.0)
        out["scatterAnisotropy"] = f("scatterAnisotropy")
        # clearcoat (:325-347): the normal from pbrMat.T / B before the tangent update
        out["clearcoat"] = f("clearcoatFactor") * tex("clearcoatTexture", one)[0][:, 0]
        ccr = f("clearcoatRoughness") * tex("clearcoatRoughnessTexture", one)[0][:, 1]
        cn, has_cn = tex("clearcoatNormalTexture", one)
        cv = cn[:, :3] * 2.0 - 1.0
        out["Nc"] = np.where(has_cn[:, None], _norm(T * cv[:, 0:1] + B * cv[:, 1:2] + pN * cv[:, 2:3]), pN)
        out["clearcoatRoughness"] = np.maximum(ccr, 0.001)
        # iridescence (:349-365)
        irid = f("iridescenceFactor") * tex("iridescenceTexture", one)[0][:, 0]
        it, has_it = tex("iridescenceThicknessTexture", one)
        lo, hi = f("iridescenceThicknessMinimum"), f("iridescenceThicknessMaximum")
        thick = np.where(has_it, lo + (hi - lo) * it[:, 1], hi)
        m = np.where(has_it, thick, np.where(thick > 0, np.inf, -np.inf))
        pos = self._take("iridescence", m / np.maximum(1.0, np.maximum(np.abs(lo), np.abs(hi))), thick > 0, flip, near)
        taken.setdefault("iridescence", set()).update(set(pos.tolist()))
        out["iridescence"] = np.where(pos, irid, 0.0)
        out["iridescenceThickness"] = thick
        out["iridescenceIor"] = f("iridescenceIor")
        # anisotropy (:367-397)
        strength = f("anisotropyStrength")
        aniso = strength > 0
        at, has_at = tex("anisotropyTexture", one)
        dx, dy = at[:, 0] * 2.0 - 1.0, at[:, 1] * 2.0 - 1.0
        ln = np.hypot(dx, dy)
        with np.errstate(invalid="ignore", divide="ignore"):
            dirx = np.where(has_at, dx / ln, 1.0)
            diry = np.where(has_at, dy / ln, 0.0)
        strength = np.where(has_at, strength * at[:, 2], strength)
        roughness[:, 0] = np.where(aniso, roughness[:, 1] + (1.0 - roughness[:, 1]) * strength * strength, roughness[:, 0])
        rot = f("anisotropyRotation", 2)
        s_, c_ = rot[:, 0], rot[:, 1]
        ax, ay = c_ * dirx + s_ * diry, c_ * diry - s_ * dirx
        pT = np.where(aniso[:, None], T * ax[:, None] + B * ay[:, None], T)
        update |= aniso
        out["roughness"] = roughness
        # tangent update (:400-407)
        nb = _norm(np.cross(pN, pT))
        m = np.where(update, _dot(B, nb), np.inf)
        with np.errstate(invalid="ignore"):
            sgn = np.sign(m)
        close = np.abs(m) < EPS["bitangentSign"]
        near["bitangentSign"] = near.get("bitangentSign", np.zeros(n, bool)) | close
        sgn = np.where(close & self._flips("bitangentSign", flip), -sgn, sgn)
        pB = np.where(update[:, None], nb * sgn[:, None], B)
        pT = np.where(update[:, None], _norm(np.cross(pB, pN) * sgn[:, None]), pT)
        out.update(N=pN, T=pT, B=pB, Ng=Ng)
        # sheen (:409-424)
        out["sheenColor"] = f("sheenColorFactor", 3) * tex("sheenColorTexture", one)[0][:, :3]
        out["sheenRoughness"] = np.maximum(MICROFACET_MIN_ROUGHNESS, f("sheenRoughnessFactor") * tex("sheenRoughnessTexture", one)[0][:, 3])
        # dispersion, diffuse transmission, retroreflection (:426-454)
        out["dispersion"] = f("dispersion")
        out["diffuseTransmissionFactor"] = f("diffuseTransmissionFactor") * tex("diffuseTransmissionTexture", one)[0][:, 3]
        out["diffuseTransmissionColor"] = f("diffuseTransmissionColor", 3) * tex("diffuseTransmissionColorTexture", one)[0][:, :3]
        out["retroreflection"] = f("retroreflectionFactor") * tex("retroreflectionTexture", one)[0][:, 0]
        return out

    # ---- one hit ------------------------------------------------------------------------------------------------------
    def evaluate(self, rec_in, hits, flip=None, only=None):
        """rec_in: the shade_io input records [n, 16]; hits: (node, tri, u, v, t) of the implementation's closest hits (hits
        only).  Returns (fields: dict name -> float64 [n] or [n, w], near: dict branch -> bool [n], taken: dict branch ->
        set of decisions taken)."""
        rec_in = np.asarray(rec_in, np.float32)
        node, tri, u, v, t = hits
        n = len(node)
        flip = np.zeros(n, bool) if flip is None else np.asarray(flip, bool)
        self._only = only
        near = {"any": np.zeros(n, bool)}
        taken = {}
        ray_dir = rec_in[:, 4:7].astype(np.float64)
        H = self.hit_state(node, tri, np.asarray(u, np.float32), np.asarray(v, np.float32), ray_dir, flip, near, taken)
        # rayConeWorldFootprint (unpinned) and the gradient of SampleGrad (gltf_pathtrace.slang:164,196)
        width = rec_in[:, 9].astype(np.float64) + rec_in[:, 10].astype(np.float64) * np.asarray(t, np.float64)
        foot = width / np.maximum(np.abs(_dot(H["geonrm"], -ray_dir)), 1e-3)
        H["texGrad"] = foot * H["texelDensity"] * rec_in[:, 11].astype(np.float64)
        M = self.material(node, H, rec_in[:, 8] != 0, H["texGrad"], flip, near, taken)
        H.update(M)
        near["any"] = np.logical_or.reduce([near[k] for k in near])
        return H, near, taken
