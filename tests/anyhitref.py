"""Float64 model of the any-hit loops of Trace and TraceShadow, for the any-hit tests.

Restated from the reference shaders, reading the scene description (vk_gltf_renderer_b200.scene.Scene) and nothing of either
implementation:
  Trace / TraceShadow            shaders/raytracer_interface.h.slang:69-179 (RayQuery: closest rays cull back faces, shadow
                                 rays use RAY_FLAG_NONE; opaque triangles commit, non-opaque ones draw one rand() each)
  getOpacity                     shaders/pathtrace_functions.h.slang:189-238
  getShadowTransmission          shaders/pathtrace_functions.h.slang:245-343
  instance flags                 src/gltf_scene_rtx.cpp:271-295 (opaque: no transmission, no diffuse transmission, OPAQUE alpha
                                 mode; culling disabled for double-sided, thick or transmissive materials)
  rand()                         PCG (state * 747796405 + 2891336453, RXS-M-XS output) -> k * 2^-23 (the 23-bit mantissa trick)

The reference leaves the order in which RayQuery returns candidates to the implementation.  Two things follow from the shaders
alone and are checked without any order: the probabilities (`closest_expectation`, `shadow_expectation`) and, given an order,
the outcome of one ray.  The renderer pins the order to (t, triangle id) front to back, so `replay` takes the draws of a ray's
seed in t order; crossings at bit-identical t are a tie group whose members the tests treat as interchangeable (equal opacity).

Everything is float64 except what the shaders' inputs are: fp32 vertices, matrices, factors and 8-bit texels.  A ray is
flagged (excluded from the exact checks) where fp32 may decide otherwise: within 1e-6 of a crossed triangle's edge, of tmin or
tmax, of another crossing's t (unless bit-identical), and where a draw or the MASK cutoff lies within the opacity's error bound.
"""
import numpy as np

import texref as tr

GRID_BITS = 23
GRID = 2.0 ** -GRID_BITS
MIN_TRANSMISSION = 0.01
EDGE_EPS = 1e-6
TIE_EPS = 1e-6
BARY_EPS = 3e-6            # fp32 barycentrics of the device's and the oracle's triangle test, relative to the triangle
_M32 = 0xFFFFFFFF
_LCG_A, _LCG_C = 747796405, 2891336453
_LCG_A_INV = pow(_LCG_A, -1, 1 << 32)
_RXS_M = 277803737
_RXS_M_INV = pow(_RXS_M, -1, 1 << 32)


# ---- rand(): PCG on the 2^-23 grid ---------------------------------------------------------------------------------------
def pcg(state):
    """one rand(): (next state, draw as an integer k, the draw being k * 2^-23); uint64 arrays holding 32-bit values"""
    state = np.asarray(state, np.uint64)
    s = (state * np.uint64(_LCG_A) + np.uint64(_LCG_C)) & np.uint64(_M32)
    word = (((s >> ((s >> np.uint64(28)) + np.uint64(4))) ^ s) * np.uint64(_RXS_M)) & np.uint64(_M32)
    out = ((word >> np.uint64(22)) ^ word) & np.uint64(_M32)
    return s, out >> np.uint64(9)


def draws(seeds, n):
    """the first n draws of each seed: float64 [len(seeds), n] (exact multiples of 2^-23)"""
    s = np.asarray(seeds, np.uint64)
    out = np.empty((len(s), n), np.float64)
    for i in range(n):
        s, k = pcg(s)
        out[:, i] = k.astype(np.float64) * GRID
    return out


def steps_between(seed_in, seed_out, max_steps=512):
    """how many rand() calls take each seed_in to seed_out (the LCG state is the seed); -1 where none up to max_steps does"""
    s = np.asarray(seed_in, np.uint64).copy()
    target = np.asarray(seed_out, np.uint64)
    out = np.full(len(s), -1, np.int64)
    for k in range(max_steps + 1):
        hit = (out < 0) & (s == target)
        out[hit] = k
        if (out >= 0).all():
            break
        s = (s * np.uint64(_LCG_A) + np.uint64(_LCG_C)) & np.uint64(_M32)
    return out


def seed_for_first_draw(k):
    """a seed whose first rand() is exactly k * 2^-23 (the PCG output permutation inverted)"""
    out = (int(k) << 9) & _M32
    word = out ^ (out >> 22)                       # (w >> 22) ^ w: the top 22 bits pass, one step restores the rest
    x = (word * _RXS_M_INV) & _M32
    shift = (x >> 28) + 4                          # the top 4 bits of the state survive its own xorshift
    s = x
    for _ in range(8):
        s = x ^ (s >> shift)
    return ((s - _LCG_C) * _LCG_A_INV) & _M32


def p_closest(a):
    """P(rand() <= a) on the grid: min(1, (floor(a 2^23) + 1) 2^-23), 0 for a < 0"""
    a = np.asarray(a, np.float64)
    return np.clip((np.floor(a * 2.0 ** GRID_BITS) + 1.0) * GRID, 0.0, 1.0)


def p_shadow(a):
    """P(rand() < a) on the grid: min(1, ceil(a 2^23) 2^-23)"""
    a = np.asarray(a, np.float64)
    return np.clip(np.ceil(a * 2.0 ** GRID_BITS) * GRID, 0.0, 1.0)


def schlick_fresnel(ior, c):
    f0 = ((ior - 1.0) / (ior + 1.0)) ** 2
    return f0 + (1.0 - f0) * (1.0 - c) ** 5


def _glm(m16):
    return np.asarray(m16, np.float64).reshape(4, 4).T


def _unorm_alpha(colors):
    return (np.asarray(colors, np.uint32) >> np.uint32(24)).astype(np.float64) / 255.0


def _by_node(mask, node):
    """(render node, (rows, columns) of its crossings in mask), one node at a time"""
    rows, cols = np.nonzero(mask)
    nodes = node[rows, cols]
    order = np.argsort(nodes, kind="stable")
    ids, start = np.unique(nodes[order], return_index=True)
    for i, a, b in zip(ids, start, list(start[1:]) + [len(order)]):
        o = order[a:b]
        yield int(i), (rows[o], cols[o])


# ---- the scene ---------------------------------------------------------------------------------------------------------
class SceneModel:
    """World-space triangles of a scene's visible render nodes, with what the any-hit loops read of each."""

    def __init__(self, scn):
        self.scn = scn
        v0, v1, v2, node, tri, nocull, opaque, mirror, nrm = [], [], [], [], [], [], [], [], []
        for i, rn in enumerate(scn.render_nodes):
            if not rn.get("visible", True):
                continue
            p = scn.render_prims[rn["renderPrimID"]]
            m = scn.materials[max(0, rn["materialID"])]
            M, W2O = _glm(rn["objectToWorld"]), _glm(rn["worldToObject"])
            P = p["positions"].astype(np.float64)
            idx = p["indices"].astype(np.int64)
            W = P @ M[:3, :3].T + M[:3, 3]
            v0.append(W[idx[:, 0]]), v1.append(W[idx[:, 1]]), v2.append(W[idx[:, 2]])
            n_obj = np.cross(P[idx[:, 1]] - P[idx[:, 0]], P[idx[:, 2]] - P[idx[:, 0]])
            n_obj /= np.linalg.norm(n_obj, axis=1, keepdims=True)
            n_w = n_obj @ W2O[:3, :3]                          # mul(worldToObject, n): the normal by the inverse transpose
            nrm.append(n_w / np.linalg.norm(n_w, axis=1, keepdims=True))
            T = len(idx)
            node.append(np.full(T, i)), tri.append(np.arange(T))
            nocull.append(np.full(T, m.doubleSided == 1 or m.thicknessFactor > 0 or m.transmissionFactor > 0))
            opaque.append(np.full(T, m.transmissionFactor == 0 and m.alphaMode == 0 and m.diffuseTransmissionFactor == 0))
            mirror.append(np.full(T, np.linalg.det(M[:3, :3]) < 0))
        cat = np.concatenate
        self.v0, self.v1, self.v2, self.normal = cat(v0), cat(v1), cat(v2), cat(nrm)
        self.node, self.tri = cat(node), cat(tri)
        self.nocull, self.opaque, self.mirror = cat(nocull), cat(opaque), cat(mirror)
        self.tex = [tr.TexRef([t["rgba8"]], t["srgb"], t["wrapS"], t["wrapT"], t["magFilter"], t["minFilter"]) for t in scn.textures]

    # -- crossings -------------------------------------------------------------------------------------------------------
    def crossings(self, rays, shadow, chunk=2048):
        """Every crossing of every ray in [tmin, tmax] (shadow rays: no culling), sorted by t.  Returns a dict of
        [R, K] arrays t, j (model triangle, -1 past the count), u, v, and n [R], flag [R]."""
        rays = np.asarray(rays, np.float32)
        e1, e2 = self.v1 - self.v0, self.v2 - self.v0
        parts = []
        for a in range(0, len(rays), chunk):
            r = rays[a:a + chunk].astype(np.float64)
            o, d = r[:, 0:3], r[:, 4:7]
            tmin = r[:, 3]                                    # RayDesc.TMin, for shadow rays too
            tmax = r[:, 7]
            # Moeller-Trumbore, one [rays, triangles] array per component
            D = [d[:, i:i + 1] for i in range(3)]
            A, B = [e1[None, :, i] for i in range(3)], [e2[None, :, i] for i in range(3)]
            pv = [D[1] * B[2] - D[2] * B[1], D[2] * B[0] - D[0] * B[2], D[0] * B[1] - D[1] * B[0]]
            det = A[0] * pv[0] + A[1] * pv[1] + A[2] * pv[2]
            with np.errstate(divide="ignore", invalid="ignore"):
                inv = 1.0 / det
                tv = [o[:, i:i + 1] - self.v0[None, :, i] for i in range(3)]
                u = (tv[0] * pv[0] + tv[1] * pv[1] + tv[2] * pv[2]) * inv
                qv = [tv[1] * A[2] - tv[2] * A[1], tv[2] * A[0] - tv[0] * A[2], tv[0] * A[1] - tv[1] * A[0]]
                v = (D[0] * qv[0] + D[1] * qv[1] + D[2] * qv[2]) * inv
                t = (B[0] * qv[0] + B[1] * qv[1] + B[2] * qv[2]) * inv
            w = 1.0 - u - v
            front = np.where(self.mirror[None], det < 0, det > 0)      # facing is the object-space winding
            live = (det != 0) & (shadow | self.nocull[None] | front)
            in_t = live & (t >= tmin[:, None]) & (t <= tmax[:, None])
            bmin = np.minimum(np.minimum(u, v), w)
            hit = in_t & (bmin >= 0)
            scale = np.maximum(np.abs(t), 1.0)
            flag = (in_t & (np.abs(bmin) < EDGE_EPS)).any(1)
            near_lim = live & (bmin > -EDGE_EPS) & ((np.abs(t - tmin[:, None]) <= EDGE_EPS * scale)
                                                     | (np.abs(t - tmax[:, None]) <= EDGE_EPS * scale))
            flag |= near_lim.any(1)
            n = hit.sum(1)
            K = max(int(n.max()) if len(n) else 0, 1)
            key = np.where(hit, t, np.inf)
            order = np.lexsort((np.broadcast_to(np.arange(t.shape[1]), t.shape), key), axis=1)[:, :K]
            take = lambda x: np.take_along_axis(x, order, 1)
            ts, us, vs = take(key), take(u), take(v)
            js = np.where(np.isfinite(ts), order, -1)
            with np.errstate(invalid="ignore"):
                dt = np.diff(ts, axis=1)
                tie = (dt > 0) & (dt < TIE_EPS * np.maximum(ts[:, 1:], 1e-30))
            flag |= tie.any(1)
            parts.append((ts, js, us, vs, n, flag))
        K = max(p[0].shape[1] for p in parts)
        pad = lambda x, fill: np.pad(x, ((0, 0), (0, K - x.shape[1])), constant_values=fill)
        out = dict(t=np.concatenate([pad(p[0], np.inf) for p in parts]), j=np.concatenate([pad(p[1], -1) for p in parts]),
                   u=np.concatenate([pad(p[2], 0.0) for p in parts]), v=np.concatenate([pad(p[3], 0.0) for p in parts]),
                   n=np.concatenate([p[4] for p in parts]), flag=np.concatenate([p[5] for p in parts]))
        out["valid"] = out["j"] >= 0
        return out

    # -- getOpacity --------------------------------------------------------------------------------------------------------
    def _texel_alpha(self, slot, prim, idx, bary, channel):
        """level-0 channel of texture-info `slot` at the interpolated TEXCOORD_n, and its error bound from the fp32 uv"""
        scn = self.scn
        ti = scn.texture_infos[slot]
        tex = self.tex[ti.index]
        uvs = prim["uv1" if ti.texCoord else "uv0"]
        if uvs is None:
            uvs = np.zeros((len(prim["positions"]), 2), np.float32)
        U = uvs.astype(np.float64)[idx]                           # [n, 3, 2]
        uv = np.einsum("nk,nkc->nc", bary, U)
        span = np.abs(U - U[:, :1]).max((1, 2)) + np.abs(U).max((1, 2)) + 1.0
        eps = BARY_EPS * span[:, None] * np.array([tex.w0, tex.h0], np.float64)   # texel-space error bound per axis
        val = tex.sample_level(0, uv.astype(np.float32), tex.mag_linear)[:, channel]
        xy = uv.astype(np.float32) * np.array([tex.w0, tex.h0], np.float32)
        if tex.mag_linear:
            err = eps.max(1)                                      # a texel-to-texel step is at most 1 per texel
        else:
            near = np.abs(xy - np.round(xy)) < eps               # NEAREST: a texel edge within reach decides nothing
            err = np.where(near.any(1), np.inf, 0.0)
        return val, err

    def opacity(self, cr):
        """getOpacity of every crossing: a [R, K] (1 for opaque triangles), its error bound, opaque [R, K]"""
        scn = self.scn
        R, K = cr["j"].shape
        a = np.ones((R, K))
        err = np.zeros((R, K))
        valid = cr["valid"]
        j = np.where(valid, cr["j"], 0)
        opaque = valid & self.opaque[j]
        node = self.node[j]
        for i, sel in _by_node(valid & ~opaque, node):
            rn = scn.render_nodes[i]
            m = scn.materials[max(0, rn["materialID"])]
            if m.alphaMode == 0:
                continue                                          # transmissive, OPAQUE alpha mode: opacity 1
            prim = scn.render_prims[rn["renderPrimID"]]
            idx = prim["indices"].astype(np.int64)[self.tri[j[sel]]]
            u, v = cr["u"][sel], cr["v"][sel]
            bary = np.stack([1.0 - u - v, u, v], 1)
            spec_gloss = m.pbrModel == 1
            x = np.full(len(u), float(m.pbrDiffuseFactor[3] if spec_gloss else m.pbrBaseColorFactor[3]))
            e = np.zeros(len(u))
            slot = m.pbrDiffuseTexture if spec_gloss else m.pbrBaseColorTexture
            if slot > 0:
                ta, te = self._texel_alpha(slot, prim, idx, bary, 3)
                e = e + x * te
                x = x * ta
            if prim["colors"] is not None:
                x = x * np.einsum("nk,nk->n", bary, _unorm_alpha(prim["colors"])[idx])
            e = e + 1e-6
            if m.alphaMode == 1:
                near = np.abs(x - float(m.alphaCutoff)) <= e
                x = np.where(x >= float(m.alphaCutoff), 1.0, 0.0)
                e = np.where(near, np.inf, 0.0)
            elif slot <= 0 and prim["colors"] is None:
                e = np.zeros(len(u))                              # the fp32 factor itself: exact
            a[sel], err[sel] = x, e
        return a, err, opaque

    # -- getShadowTransmission -----------------------------------------------------------------------------------------------
    def transmission(self, cr, dirs):
        """the per-crossing factor of getShadowTransmission without the Beer term: c [R, K, 3], and per crossing the material's
        thickness flag and absorption coefficient [R, K, 3] (used inside a thick material)"""
        scn = self.scn
        R, K = cr["j"].shape
        c = np.zeros((R, K, 3))
        thick = np.zeros((R, K), bool)
        absorb = np.zeros((R, K, 3))
        valid = cr["valid"]
        j = np.where(valid, cr["j"], 0)
        node = self.node[j]
        d = np.asarray(dirs, np.float32).astype(np.float64)
        for i, sel in _by_node(valid, node):
            rn = scn.render_nodes[i]
            m = scn.materials[max(0, rn["materialID"])]
            tf = float(m.transmissionFactor)
            if tf <= MIN_TRANSMISSION:
                continue
            assert max(m.multiscatterColorFactor[:3]) == 0, "the model restates thick materials without volume scattering"
            rows = sel[0]
            cos = np.abs(np.sum(d[rows] * self.normal[j[sel]], 1))
            cur = np.asarray(m.pbrBaseColorFactor[:3], np.float64)[None] * tf * (1.0 - schlick_fresnel(float(m.ior), cos))[:, None]
            rough, metal = np.full(len(cos), float(m.pbrRoughnessFactor)), np.full(len(cos), float(m.pbrMetallicFactor))
            if m.pbrMetallicRoughnessTexture > 0:
                prim = scn.render_prims[rn["renderPrimID"]]
                idx = prim["indices"].astype(np.int64)[self.tri[j[sel]]]
                bary = np.stack([1.0 - cr["u"][sel] - cr["v"][sel], cr["u"][sel], cr["v"][sel]], 1)
                rough = rough * self._texel_alpha(m.pbrMetallicRoughnessTexture, prim, idx, bary, 1)[0]
                metal = metal * self._texel_alpha(m.pbrMetallicRoughnessTexture, prim, idx, bary, 2)[0]
            att = (1.0 - metal) * (0.65 + 0.35 * (1.0 - rough * rough))
            c[sel] = cur * att[:, None]
            if m.thicknessFactor > 0:
                thick[sel] = True
                absorb[sel] = (-np.log(np.maximum(np.asarray(m.attenuationColor[:3], np.float64), 0.001))
                               / max(float(m.attenuationDistance), 0.001))[None]
        return c, thick, absorb

    def layer_of(self, cr):
        """render node of every crossing ([R, K], -1 past the count)"""
        return np.where(cr["valid"], self.node[np.where(cr["valid"], cr["j"], 0)], -1)


# ---- one ray, given its seed -------------------------------------------------------------------------------------------
def _candidates(cr, opaque):
    """closest rays: the non-opaque crossings in front of the nearest opaque one, and the index of that opaque one (-1: none)"""
    valid = cr["valid"]
    first_opq = np.where((valid & opaque).any(1), np.argmax(valid & opaque, 1), -1)
    K = valid.shape[1]
    before = np.arange(K)[None] < np.where(first_opq >= 0, first_opq, K)[:, None]
    return valid & ~opaque & before, first_opq


def replay_closest(cr, a, err, opaque, seeds):
    """Trace with the draws of each seed in t order: hit index into the crossings (-1: miss), draws used, flag (a draw within
    the opacity's error bound)"""
    cand, first_opq = _candidates(cr, opaque)
    R, K = cand.shape
    U = draws(seeds, K)
    rank = np.cumsum(cand, 1) - 1
    u = np.take_along_axis(U, np.maximum(rank, 0), 1)
    acc = cand & (u <= a)
    any_acc = acc.any(1)
    first = np.argmax(acc, 1)
    hit = np.where(any_acc, first, first_opq)
    used = np.where(any_acc, rank[np.arange(R), first] + 1, cand.sum(1))
    drawn = cand & (rank < used[:, None])
    flag = (drawn & (np.abs(u - a) < err)).any(1)
    return hit, used, flag


def replay_shadow(cr, a, err, opaque, c, thick, absorb, seeds):
    """TraceShadow with the draws of each seed in t order: transmission [R, 3], draws used, flag"""
    valid = cr["valid"]
    R, K = valid.shape
    U = draws(seeds, K)
    blocked = (valid & opaque).any(1)
    T = np.ones((R, 3))
    alive = ~blocked
    used = np.zeros(R, np.int64)
    prev = np.zeros(R)
    inside = np.zeros(R, bool)
    flag = np.zeros(R, bool)
    for k in range(K):
        live = alive & valid[:, k]
        u = U[np.arange(R), np.minimum(used, K - 1)]
        acc = live & (u < a[:, k])
        flag |= live & (np.abs(u - a[:, k]) < err[:, k])
        used += live
        seg = np.maximum(0.0, cr["t"][:, k] - prev)
        cur = c[:, k].copy()
        beer = acc & thick[:, k] & inside
        cur[beer] *= np.exp(-seg[beer, None] * absorb[beer, k])
        inside ^= acc & thick[:, k]
        prev = np.where(acc, cr["t"][:, k], prev)
        T[acc] *= cur[acc]
        m = T.max(1)
        flag |= acc & (np.abs(m - MIN_TRANSMISSION) <= 1e-5 * MIN_TRANSMISSION)
        dead = acc & (m <= MIN_TRANSMISSION)
        T[dead] = 0.0
        alive &= ~dead
    T[blocked] = 0.0
    return T, used, flag


# ---- order-free expectations -------------------------------------------------------------------------------------------
def closest_expectation(cr, a, opaque):
    """P(stop at crossing k) [R, K], P(opaque hit) [R], P(miss) [R], E[draws] [R], Var[draws] [R]"""
    cand, first_opq = _candidates(cr, opaque)
    p = np.where(cand, p_closest(a), 0.0)
    reach = np.cumprod(np.concatenate([np.ones((len(p), 1)), 1.0 - p[:, :-1]], 1), 1)   # prod_{j<k} (1 - p_j)
    stop = np.where(cand, p * reach, 0.0)
    none = np.prod(1.0 - p, 1)
    p_opq = np.where(first_opq >= 0, none, 0.0)
    p_miss = np.where(first_opq >= 0, 0.0, none)
    rank = np.cumsum(cand, 1)                                     # draws used when stopping at k
    e_d = (stop * rank).sum(1) + none * cand.sum(1)
    e_d2 = (stop * rank ** 2).sum(1) + none * cand.sum(1) ** 2
    return stop, p_opq, p_miss, e_d, e_d2 - e_d ** 2


def shadow_expectation(cr, a, opaque, c, thick, absorb, max_enum=12):
    """E[T] [R, 3], E[T^2] [R, 3], E[draws] [R], E[draws^2] [R] by enumerating the accepted subsets front to back (stochastic
    crossings only: p = 0 or 1 does not branch); rays whose layers stop the ray outright (c = 0) in closed form"""
    valid = cr["valid"]
    R, K = valid.shape
    p = np.where(valid, p_shadow(a), 0.0)
    blocked = (valid & opaque).any(1)
    ET, ET2 = np.zeros((R, 3)), np.zeros((R, 3))
    ED, ED2 = np.zeros(R), np.zeros(R)
    black = ~blocked & (~valid | (c.max(2) <= MIN_TRANSMISSION)).all(1)
    # closed form: the first accepted crossing ends the ray with T = 0
    reach = np.cumprod(np.concatenate([np.ones((R, 1)), 1.0 - p[:, :-1]], 1), 1)
    none = np.prod(1.0 - p, 1)
    stop = np.where(valid, p * reach, 0.0)
    k1 = np.arange(1, K + 1)[None]
    n = valid.sum(1)
    ET[black] = none[black, None]
    ET2[black] = none[black, None]
    ED[black] = ((stop * k1).sum(1) + none * n)[black]
    ED2[black] = ((stop * k1 ** 2).sum(1) + none * n ** 2)[black]
    # the rest: every accept / reject pattern of a ray's stochastic crossings (0 < p < 1) is one state, bit b of the state
    # deciding the b-th of them; crossings with p = 0 or 1 decide the same in every state
    rest = np.nonzero(~blocked & ~black)[0]
    if len(rest):
        stoch = valid & (p > 0) & (p < 1)
        bits = stoch[rest].sum(1)
        assert bits.max() <= max_enum, f"{bits.max()} stochastic crossings: beyond the enumeration"
        S = 1 << int(bits.max())
        chunk = max(1, (1 << 20) // S)
        for a0 in range(0, len(rest), chunk):
            rr = rest[a0:a0 + chunk]
            R2 = len(rr)
            st = np.arange(S)[None]
            q = (st < (1 << bits[a0:a0 + chunk])[:, None]).astype(np.float64)
            T = np.ones((R2, S, 3))
            prev = np.zeros((R2, S))
            inside = np.zeros((R2, S), bool)
            alive = np.ones((R2, S), bool)
            dr = np.zeros((R2, S))
            rank = np.cumsum(stoch[rr], 1) - 1
            for k in range(K):
                pk = p[rr, k][:, None]
                live = alive & valid[rr, k][:, None]
                bit = ((st >> np.maximum(rank[:, k], 0)[:, None]) & 1) == 1
                acc = live & np.where(stoch[rr, k][:, None], bit, pk >= 1.0)
                q = np.where(live & stoch[rr, k][:, None], q * np.where(bit, pk, 1.0 - pk), q)
                dr += live
                cur = np.broadcast_to(c[rr, k][:, None, :], (R2, S, 3)).copy()
                beer = acc & thick[rr, k][:, None] & inside
                seg = np.maximum(0.0, cr["t"][rr, k][:, None] - prev)
                cur[beer] *= np.exp(-seg[beer][:, None] * np.broadcast_to(absorb[rr, k][:, None, :], (R2, S, 3))[beer])
                inside ^= acc & thick[rr, k][:, None]
                prev = np.where(acc, cr["t"][rr, k][:, None], prev)
                T = np.where(acc[..., None], T * cur, T)
                dead = acc & (T.max(2) <= MIN_TRANSMISSION)
                T[dead] = 0.0
                alive &= ~dead
            ET[rr] = np.einsum("rs,rsc->rc", q, T)
            ET2[rr] = np.einsum("rs,rsc->rc", q, T * T)
            ED[rr] = (q * dr).sum(1)
            ED2[rr] = (q * dr * dr).sum(1)
    return ET, ET2, ED, ED2


def identical_stack(n, p, c):
    """E[T] of n identical non-thick layers (acceptance p, factor c [3]) by a DP over the number of accepted layers: after k
    acceptances T = c^k, and the ray ends with 0 at the first k where max(c^k) <= 0.01"""
    from scipy.stats import binom
    c = np.asarray(c, np.float64)
    out = np.zeros(3)
    for k in range(n + 1):
        if any((c ** m).max() <= MIN_TRANSMISSION for m in range(1, k + 1)):
            break
        out += binom.pmf(k, n, p) * c ** k
    return out


def monte_carlo_transmission(p, c, t, thick, absorb, trials, rng):
    """numpy Monte Carlo of one ray's TraceShadow: acceptance drawn per crossing front to back; returns E[T] [3]"""
    K = len(p)
    acc = rng.random((trials, K)) < p[None]
    T = np.ones((trials, 3))
    prev = np.zeros(trials)
    inside = np.zeros(trials, bool)
    alive = np.ones(trials, bool)
    for k in range(K):
        ak = acc[:, k] & alive
        cur = np.broadcast_to(c[k], (trials, 3)).copy()
        beer = ak & thick[k] & inside
        cur[beer] *= np.exp(-np.maximum(0.0, t[k] - prev[beer])[:, None] * absorb[k][None])
        inside ^= ak & thick[k]
        prev = np.where(ak, t[k], prev)
        T[ak] *= cur[ak]
        dead = ak & (T.max(1) <= MIN_TRANSMISSION)
        T[dead] = 0.0
        alive &= ~dead
    return T.mean(0)
