"""Float64 expectation of the path tracer's estimator at one shading point, for the tests that render it.

The expectation is that of the estimator as oracle/pt_oracle.cpp and csrc/shade.cuh / csrc/b200pt.cu define it, following the
reference (shaders/pathtrace_functions.h.slang, shaders/gltf_pathtrace.slang): the bilinearly filtered environment alpha is
the pdf in every MIS weight, the light / environment MIS of sampleLights ignores the BSDF, and a BSDF-sampled ray that leaves
the scene is weighted against the environment only.  Where that differs from the rendering equation the difference is
computed here (`rendering_equation`), not corrected.

Conventions restated (line numbers: shade.cuh / b200pt.cu on the device, pt_oracle.cpp in the oracle, the reference):
  - lat-long map: uv = (atan2(z, x) / 2pi + 1/2, asin(-y) / pi + 1/2) (bsdf.cuh:813, bsdf.h:890); the sampler draws
    phi = 2pi u - pi and cos(theta) = y linearly between the texel's row edges (shade.cuh:624-655, pt_oracle.cpp:392-422,
    nvshaders hdr_env_sampling).
  - `envRotation`: a sampled direction is turned by +rotation about +y, a looked-up direction by -rotation
    (shade.cuh:784-792, b200pt.cu:729, :1067; pathtrace_functions.h.slang:440, 444, 475).
  - lookup: bilinear, level 0, texel centres at half-integers, repeat in u, clamp in v (shade.cuh:605, pt_oracle.cpp:372).
  - alpha: max(r, g, b) / sum_i (area_i max_i), area_i = (cos theta0 - cos theta1) 2pi / W (pt_oracle.cpp:342-369).
  - technique probabilities 0.5 / 0.5 (shade.cuh:740, pathtrace_functions.h.slang:357-378); a light is chosen with
    1 / numLights and its radiance divided by selectionPdf * lightWeight (shade.cuh:763-806, :410-412 of the reference);
    the light / environment MIS pdfSum = lightWeight pdf_light + envWeight envPdf (:455-457).
  - NEE vs BSDF: pdfSum / (pdfSum + pdf_bsdf), 1 for a Dirac light (b200pt.cu:963, gltf_pathtrace.slang:344); the
    environment hit of a BSDF-sampled ray: pdf_bsdf / (pdf_bsdf + envWeight envPdf) (b200pt.cu:728-737, :1072-1079,
    pathtrace_functions.h.slang:483-491).
  - singleLightContribution (shade.cuh:667, pt_oracle.cpp:1393; nvshaders light_contrib, external).
All sums are float64.  BSDF values come from tests/bsdfref.py.
"""
import numpy as np

import bsdfref as R

TWO_PI = 2.0 * np.pi


# ---- environment ---------------------------------------------------------------------------------------------------------
def rotate_y(d, a):
    """rotate(v, (0, 1, 0), a) of bsdf.h:897: Rodrigues about +y"""
    c, s = np.cos(a), np.sin(a)
    x, y, z = d[..., 0], d[..., 1], d[..., 2]
    return np.stack([x * c + z * s, y, z * c - x * s], -1)


def dir_to_uv(d):
    """getSphericalUv"""
    return (np.arctan2(d[..., 2], d[..., 0]) / TWO_PI + 0.5, np.arcsin(np.clip(-d[..., 1], -1, 1)) / np.pi + 0.5)


def phi_cos_to_dir(phi, ct):
    """the sampler's direction for phi = 2pi u - pi and cos(theta)"""
    st = np.sqrt(np.maximum(0.0, 1.0 - ct * ct))
    return np.stack([np.cos(phi) * st, ct, np.sin(phi) * st], -1)


class Env:
    """One lat-long environment: the stored texels (rgb and alpha as the renderer keeps them), the alias table the oracle
    built, and the float64 quantities the estimator's expectation needs."""

    def __init__(self, rgba, alias, q):
        self.rgba = np.asarray(rgba, np.float64)
        self.h, self.w = self.rgba.shape[:2]
        self.alias = np.asarray(alias, np.int64)
        self.q = np.asarray(q, np.float64)
        ct = np.cos(np.arange(self.h + 1) * (np.pi / self.h))
        self.cos_edges = ct
        self.row_area = (ct[:-1] - ct[1:]) * (TWO_PI / self.w)

    @classmethod
    def from_oracle(cls, oracle):
        return cls(*oracle.get_environment())

    def texel_prob(self):
        """P(i) = (q_i + sum_{alias_j = i} (1 - q_j)) / N: the probability that environmentSample picks texel i (xi.x picks
        j uniformly, xi.y keeps j with probability q_j, else takes alias_j)"""
        n = self.w * self.h
        keep = np.clip(self.q, 0.0, 1.0)
        p = np.bincount(np.arange(n), keep, n) + np.bincount(self.alias, 1.0 - keep, n)
        return (p / n).reshape(self.h, self.w)

    def ideal_prob(self):
        """importance_i / sum importance with the float64 importance area_i max(r, g, b)"""
        imp = self.row_area[:, None] * self.rgba[..., :3].max(-1)
        return imp / imp.sum()

    def density(self, prob=None):
        """density per unit solid angle of the sampled direction, constant per texel: P(i) / area_i"""
        prob = self.texel_prob() if prob is None else prob
        return prob / self.row_area[:, None]

    def lookup(self, d):
        """sampleEnvTex(getSphericalUv(d)) in float64: rgba [n, 4]"""
        u, v = dir_to_uv(d)
        x, y = u * self.w - 0.5, v * self.h - 0.5
        x0, y0 = np.floor(x), np.floor(y)
        fx, fy = (x - x0)[:, None], (y - y0)[:, None]
        x0, y0 = x0.astype(np.int64), y0.astype(np.int64)

        def at(xi, yi):
            return self.rgba[np.clip(yi, 0, self.h - 1), xi % self.w]
        top = at(x0, y0) * (1 - fx) + at(x0 + 1, y0) * fx
        bot = at(x0, y0 + 1) * (1 - fx) + at(x0 + 1, y0 + 1) * fx
        return top * (1 - fy) + bot * fy

    def nodes(self, sub, rows):
        """midpoint nodes of a sub x sub grid in (phi, cos theta) inside every texel of `rows`: environment-frame directions
        [n, 3], solid-angle weights [n], texel (row, column) [n] each"""
        r = np.asarray(rows)
        k = (np.arange(sub) + 0.5) / sub
        c0, c1 = self.cos_edges[r], self.cos_edges[r + 1]
        ct = c0[:, None] + (c1 - c0)[:, None] * k[None, :]                                  # [rows, sub]
        px = (np.arange(self.w)[:, None] + k[None, :]).reshape(-1)                          # [w * sub]
        phi = px / self.w * TWO_PI - np.pi
        CT = np.repeat(ct, self.w * sub, 1).reshape(-1)
        PH = np.tile(phi, len(r) * sub)
        row = np.repeat(r, sub * self.w * sub)
        col = np.tile(np.repeat(np.arange(self.w), sub), len(r) * sub)
        wgt = np.repeat(self.row_area[r] / (sub * sub), sub * self.w * sub)
        return phi_cos_to_dir(PH, CT), wgt, row, col

    def integrate(self, fn, sub, chunk_nodes=1 << 21):
        """sum over nodes of fn(env-frame dirs, weights, row, col) -> [n, k], in row chunks"""
        per_row = self.w * sub * sub
        step = max(1, chunk_nodes // per_row)
        total = 0.0
        for r0 in range(0, self.h, step):
            d, wgt, row, col = self.nodes(sub, np.arange(r0, min(self.h, r0 + step)))
            total = total + fn(d, wgt, row, col).sum(0)
        return total


# ---- the BSDF at a shading point -------------------------------------------------------------------------------------------
class Bsdf:
    """One lobe of tests/bsdfref.py at a shading point with normal n, seen from v (both world, unit): `eval(k2)` returns
    (pdf [n], bsdf_diffuse + bsdf_glossy [n, 3]) of bsdfEvaluate; the material has this lobe only (weight 1)."""

    def __init__(self, n, v, lobe, base=(1.0, 1.0, 1.0), alpha=0.3):
        n, v = np.asarray(n, np.float64), np.asarray(v, np.float64)
        t = v - n * (v @ n)
        if np.linalg.norm(t) < 1e-9:
            t = np.cross(n, [1.0, 0, 0] if abs(n[0]) < 0.9 else [0, 1.0, 0])
        self.T = t / np.linalg.norm(t)
        self.B = np.cross(n, self.T)
        self.N = n
        theta = np.degrees(np.arccos(np.clip(v @ n, -1, 1)))
        self.rec = R.record(base=base, alpha=(alpha, alpha), metallic=1.0 if lobe == R.METAL else 0.0, specular=0.0,
                            theta=theta, phi=0.0)
        self.lobe = lobe

    def local(self, k2):
        return np.stack([k2 @ self.T, k2 @ self.B, k2 @ self.N], -1)

    def eval(self, k2):
        return R.lobe_eval(self.rec, self.local(k2), self.lobe)

    def albedo(self, nc=512, nphi=512):
        """integral of f cos over the sphere, on the lobe's own nodes (bsdfref.nodes)"""
        k2, w, _ = R.nodes(self.rec, self.lobe, nc, nphi)
        _, val = R.lobe_eval(self.rec, k2, self.lobe)
        return (w[:, None] * val).sum(0)


# ---- punctual lights -------------------------------------------------------------------------------------------------------
def smoothstep(e0, e1, x):
    t = np.clip((x - e0) / (e1 - e0), 0.0, 1.0)
    return t * t * (3.0 - 2.0 * t)


def light_contribution(light, pos):
    """singleLightContribution without the sampling: (direction to the light's centre, half angular size, intensity rgb)"""
    ldir = np.array(light.direction[:], np.float64)
    color = np.array(light.color[:], np.float64)
    if light.type == 1:
        return -ldir, 0.5 * light.angularSizeOrInvRange, color * light.intensity
    l2s = np.asarray(pos, np.float64) - np.array(light.position[:], np.float64)
    dist = np.linalg.norm(l2s)
    inc = l2s / dist
    att = 1.0
    if light.angularSizeOrInvRange > 0:
        att = np.clip(1.0 - (dist * light.angularSizeOrInvRange) ** 4, 0.0, 1.0) ** 2
    spot = 1.0
    if light.type == 2:
        spot = 1.0 - smoothstep(light.innerAngle, light.outerAngle, np.arccos(np.clip(inc @ ldir, -1, 1)))
    half = 0.0
    if light.radius > 0:
        half = np.arctan(min(light.radius / dist, 1.0))
        irr = light.intensity / light.radius ** 2 * half * half
    else:
        irr = light.intensity / dist ** 2
    return -inc, half, color * irr * spot * att


def cone_nodes(axis, half, nc, nphi):
    """midpoint nodes of the cone of half-angle `half` about `axis`, uniform in (cos theta, phi): directions and weights"""
    a = np.asarray(axis, np.float64)
    t = np.cross(a, [1.0, 0, 0] if abs(a[0]) < 0.9 else [0, 1.0, 0])
    t /= np.linalg.norm(t)
    b = np.cross(a, t)
    cmax = np.cos(half)
    ct = 1.0 - (np.arange(nc) + 0.5) / nc * (1.0 - cmax)
    ph = (np.arange(nphi) + 0.5) / nphi * TWO_PI
    C, P = np.meshgrid(ct, ph, indexing="ij")
    S = np.sqrt(1.0 - C * C)
    d = (S * np.cos(P))[..., None] * t + (S * np.sin(P))[..., None] * b + C[..., None] * a
    return d.reshape(-1, 3), np.full(nc * nphi, TWO_PI * (1.0 - cmax) / (nc * nphi))


# ---- the estimator's expectation at a shading point ------------------------------------------------------------------------
def technique_probabilities(num_lights, env_on):
    lw = 0.5 if num_lights > 0 else 0.0
    ew = 0.5 if env_on else 0.0
    tot = lw + ew
    return (lw / tot, ew / tot) if tot > 0 else (0.0, 0.0)


def expectation(bsdf, *, env=None, env_rotation=0.0, env_intensity=1.0, lights=(), pos=(0, 0, 0), sub=4, cone_n=(64, 64),
                realised=True, parts=False, env_terms=True):
    """E[radiance] of one sample whose first hit is this shading point, when every secondary ray escapes (a convex body),
    no shadow ray is blocked and the throughput after the hit is what the BSDF sampler returns:

        E = sum_technique P(technique) int (value added) (density sampled) d(omega)  +  BSDF-sampled environment hit

    env NEE       envW p_env(w) * I rgb(w) / (envW alpha(w) + pdf_b(w)) * f cos(w)        p_env = P(i) / area_i (realised)
    BSDF env hit  f cos(w) * I rgb(w) * pdf_b(w) / (pdf_b(w) + envW alpha(w))
    Dirac light   I_j f cos(w_j)
    cone light    int_cone pdf_c I_j w_le w_nee f cos,  w_le = lw pdf_c / n / (lw pdf_c / n + envW alpha),
                  w_nee = pdfSum / (pdfSum + pdf_b),  pdfSum = lw pdf_c / n + envW alpha
    NEE needs dot(w, n) > 0 and pdf_b(w) > 0.  `realised=False` puts alpha itself in place of p_env: the estimator as it would
    be if the sampler drew exactly the density its weights assume.  `env=None` or env_intensity 0 switches the environment
    technique off (envWeight 0 when the HDR environment has intensity 0).  env_terms=False leaves out the two environment terms
(they do not depend on `pos`) but keeps the environment's part of the light MIS.  Returns rgb, or with parts=True a dict of
terms."""
    n_l = len(lights)
    env_on = env is not None and env_intensity > 0
    lw, ew = technique_probabilities(n_l, env_on)
    out = dict(env_nee=np.zeros(3), bsdf_env=np.zeros(3), lights=np.zeros(3))
    N = bsdf.N
    if env_on and env_terms:
        dens = env.density() if realised else None

        def fn(d, wgt, row, col):
            wd = rotate_y(d, env_rotation)
            pdf_b, val = bsdf.eval(wd)
            look = env.lookup(d)
            rgb, alpha = look[:, :3] * env_intensity, look[:, 3]
            p_env = dens[row, col] if realised else alpha
            nee_ok = ((wd @ N) > 0) & (pdf_b > 0)
            with np.errstate(divide="ignore", invalid="ignore"):
                nee = np.where(nee_ok, ew * p_env / (ew * alpha + pdf_b), 0.0)
                hit = np.where(pdf_b > 0, pdf_b / (pdf_b + ew * alpha), 0.0)
            return np.concatenate([(wgt * nee)[:, None] * rgb * val, (wgt * hit)[:, None] * rgb * val], 1)
        tot = env.integrate(fn, sub)
        out["env_nee"], out["bsdf_env"] = tot[:3], tot[3:]
    for L in lights:
        wdir, half, inten = light_contribution(L, pos)
        if half == 0.0:
            pdf_b, val = bsdf.eval(wdir[None])
            if wdir @ N > 0 and pdf_b[0] > 0:
                out["lights"] += inten * val[0]
            continue
        d, wgt = cone_nodes(wdir, half, *cone_n)
        pdf_c = 1.0 / (TWO_PI * (1.0 - np.cos(half)))
        pdf_b, val = bsdf.eval(d)
        alpha = 0.0
        if env_on:
            alpha = env.lookup(rotate_y(d, -env_rotation))[:, 3]
        pl = lw * pdf_c / n_l
        psum = pl + ew * alpha
        ok = ((d @ N) > 0) & (pdf_b > 0)
        w = np.where(ok, pdf_c * (pl / psum) * (psum / (psum + pdf_b)), 0.0)
        out["lights"] += ((wgt * w)[:, None] * val).sum(0) * inten
    if parts:
        return out
    return out["env_nee"] + out["bsdf_env"] + out["lights"]


def rendering_equation(bsdf, *, env=None, env_rotation=0.0, env_intensity=1.0, lights=(), pos=(0, 0, 0), sub=4, cone_n=(64, 64)):
    """int L_in f cos over the sphere: the environment (filtered, as looked up) plus each light's cone (or Dirac value)"""
    tot = np.zeros(3)
    if env is not None and env_intensity > 0:
        def fn(d, wgt, row, col):
            pdf_b, val = bsdf.eval(rotate_y(d, env_rotation))
            return wgt[:, None] * env.lookup(d)[:, :3] * env_intensity * val
        tot += env.integrate(fn, sub)
    for L in lights:
        wdir, half, inten = light_contribution(L, pos)
        if half == 0.0:
            if wdir @ bsdf.N > 0:
                tot += inten * bsdf.eval(wdir[None])[1][0]
            continue
        d, wgt = cone_nodes(wdir, half, *cone_n)
        pdf_b, val = bsdf.eval(d)
        pdf_c = 1.0 / (TWO_PI * (1.0 - np.cos(half)))
        tot += ((wgt * pdf_c * ((d @ bsdf.N) > 0))[:, None] * val).sum(0) * inten
    return tot


# ---- closed enclosure ------------------------------------------------------------------------------------------------------
def enclosure_expectation(emission, rho, max_depth):
    """E sum_{k < K} rho^k with K = maxDepth for a closed box of single-lobe Lambertian walls (albedo rho, emission E) seen
    from inside.  pathTrace (pt_oracle.cpp:2076-2110, b200pt.cu's bounce loop, gltf_pathtrace.slang:445-485) runs bounces
    surfaceDepth = 0 .. maxDepth - 1 while surfaceDepth < maxDepth; every bounce hits a wall (the box is closed) and adds
    emissive * throughput before anything else, the last one included, so the vertex of depth k adds E rho^k for
    k = 0 .. maxDepth - 1.  The diffuse sampler returns bsdf_over_pdf = rho, so the throughput at depth k is rho^k.  Russian
    roulette runs after the bounce of depth >= 3 and divides the throughput by its continuation probability: it changes the
    variance, not the expectation.  With no light and the environment at intensity 0 there is no NEE technique (both
    technique weights are 0), and shadow rays could not leave the box anyway.  So K = maxDepth."""
    rho = np.asarray(rho, np.float64)
    return np.asarray(emission, np.float64) * sum(rho ** k for k in range(max_depth))
