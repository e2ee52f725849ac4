"""Float64 expectation of the path tracer's participating-media estimator, for the tests that render a medium box
(vk_gltf_renderer_b200.synth.synth_medium_box).

The estimator is the one oracle/pt_oracle.cpp and csrc/shade.cuh / csrc/b200pt.cu run, following the reference
(shaders/pathtrace_functions.h.slang: handleVolumeScatter, volumeScatterNEE, getShadowTransmission, the in-medium Russian
roulette of processVolumeSegment).  Restated here, independently of both:
  - coefficients: sigma_a = -ln(max(c, 0.001)) / max(d, 0.001), sigma_s = sigma_a ssa(rho_ms) with ssa the
    multiToSingleScatterAlbedo fit (gltf_material_eval.h.slang:125-129), sigma_t = sigma_a + sigma_s.  The walk keeps
    sigma_t, sigma_s and g as binary16 (round to nearest even); the shadow ray's getShadowTransmission recomputes them at
    full precision.
  - walk, when max sigma_s > 0.001: a distance is drawn with the largest extinction m = max_c sigma_t; a collision before
    the boundary scatters, with weight 1 - (sigma_t - sigma_s) / m per channel, and draws a Henyey-Greenstein direction; a
    segment that reaches the boundary is weighted exp((m - sigma_t) d).  Otherwise the segment is weighted exp(-sigma_t d).
  - at every scatter: next-event estimation with sampleLights' technique choice and light / environment MIS, a Dirac light
    rejected by pdf <= 0, the phase MIS pdfSum / (pdfSum + p_HG), and the shadow factor of getShadowTransmission:
    (1 - Schlick(ior, |cos|)) exp(-sigma_t d) and, for a scattering medium, a second exp(-m d); a shadow factor whose
    largest channel is <= 0.01 counts as 0.
  - after 64 scatters, Russian roulette at every scatter with p = min(max throughput + 0.001, 0.95).
  - the boundary: the material is a smooth dielectric (roughness 0 is clamped to 0.0014142, alpha 2e-6, a delta lobe for
    every purpose here): computeLobeWeights picks reflection with the Fresnel reflectance F(ior2 / ior1, fcos), fcos the
    roughness-adjusted cosine, else refraction (reflection under total internal reflection); both have weight 1.  A ray
    that leaves the box reaches the environment with MIS weight 1 (its BSDF pdf is ~1e10).  The BSDF value of the surface
    NEE is below 1e-10, so surfaces add no direct light.
  - surface depth: every boundary interaction is one bounce; a path runs while depth < maxDepth, and Russian roulette
    runs after every bounce of depth >= 3.
`rte` swaps parts of the estimator for the radiative-transfer behaviour, to measure the gaps; nothing asserts on it.
"""
import numpy as np

import bsdfref as R
import estref

MIN_ROUGHNESS = float(np.float32(0.0014142))
ALPHA = float(np.float32(MIN_ROUGHNESS * MIN_ROUGHNESS))
DIRAC = -1.0


def half(x):
    """round trip through IEEE binary16, round to nearest even"""
    return np.asarray(x, np.float64).astype(np.float16).astype(np.float64)


def ssa(rho):
    """multiToSingleScatterAlbedo"""
    rho = np.asarray(rho, np.float64)
    t = 4.09712 + 4.20863 * rho - np.sqrt(9.59217 + 41.6808 * rho + 17.7126 * rho * rho)
    return 1.0 - t * t


def hg_pdf(cos, g):
    d = 1.0 + g * g - 2.0 * g * cos
    return (1.0 - g * g) / (4.0 * np.pi * d * np.sqrt(d))


def hg_cos(xi, g):
    """inverse CDF of cos(theta) between the incoming and the scattered direction, forward for g > 0"""
    if g == 0.0:
        return 1.0 - 2.0 * xi
    sq = (1.0 - g * g) / (1.0 - g + 2.0 * g * xi)
    return np.clip((1.0 + g * g - sq * sq) / (2.0 * g), -1.0, 1.0)


def hg_cdf(cos, g):
    """P(cos(theta) <= cos) for the Henyey-Greenstein phase function"""
    if g == 0.0:
        return (cos + 1.0) / 2.0
    return (1.0 - g * g) / (2.0 * g) * (1.0 / np.sqrt(1.0 + g * g - 2.0 * g * cos) - 1.0 / (1.0 + g))


class Medium:
    """The coefficients of one material: `walk` (binary16, what the walk uses) and `full` (full precision, what the shadow
    ray uses), each (sigma_t [3], sigma_s [3]), and g (binary16).  `rounded=False` keeps the walk at full precision too."""

    def __init__(self, color=(1, 1, 1), distance=np.inf, ms=(0, 0, 0), g=0.0, rounded=True):
        color, ms = np.asarray(color, np.float64), np.asarray(ms, np.float64)
        with np.errstate(divide="ignore"):
            sa = -np.log(np.maximum(color, 0.001)) / max(float(distance), 0.001)
        # the walk's sigma_s is set only when a multiscatter channel is > 0; getShadowTransmission applies ssa unguarded,
        # and ssa(0) = 5.7e-6, not 0 (the fp32 fit cancels there)
        ss = sa * ssa(ms) if np.any(ms > 0) else np.zeros(3)
        self.full = (sa * (1.0 + ssa(ms)), sa * ssa(ms))
        r = half if rounded else (lambda x: np.asarray(x, np.float64))
        # the value binary16 rounds is the estimator's fp32 one: a float64 value can sit on the other side of a tie
        f = np.float32
        with np.errstate(divide="ignore"):
            sa32 = -np.log(np.maximum(color.astype(f), f(0.001))) / np.maximum(f(distance), f(0.001))
            ss32 = sa32 * ssa(ms).astype(f) if np.any(ms > 0) else np.zeros(3, f)
        self.walk = (r(sa32 + ss32), r(ss32)) if rounded else (r(sa + ss), r(ss))
        self.g = float(r(g))
        self.scatters = self.walk[1].max() > 0.001
        self.shadow_scatters = self.full[1].max() > 0.001
        self.present = self.walk[0].max() > 0 or self.walk[1].max() > 0


def offset_origin(z, up):
    """z of safeOffsetRay(p, n) for a point on the face z = const, n = (0, 0, +-1): 256 ulps along n, or 1/65536 near 0"""
    z32 = np.float32(z)
    if abs(z32) < 1.0 / 32.0:
        return float(z32 + np.float32(1.0 / 65536.0) * (1 if up else -1))
    step = 256 if (up == (z32 > 0)) else -256
    return float((np.array([z32]).view(np.int32) + step).view(np.float32)[0])


def segment(hz):
    """length of the straight segment from one z face's offset origin to the other face"""
    return offset_origin(hz, up=False) + float(np.float32(hz))


def fresnel(eta, c):
    """vectorised bsdfref.fresnel_dielectric"""
    c = np.asarray(c, np.float64)
    ct2 = 1.0 - (1.0 - c * c) / (eta * eta)
    ct = np.sqrt(np.maximum(ct2, 0.0))
    with np.errstate(divide="ignore", invalid="ignore"):
        rp = (ct - eta * c) / (ct + eta * c)
        rs = (c - eta * ct) / (c + eta * ct)
    return np.where(ct2 <= 0.0, 1.0, np.clip(0.5 * (rp * rp + rs * rs), 0.0, 1.0))


def fcos(vn):
    """the cosine computeLobeWeights gives the dielectric Fresnel term"""
    return vn + (np.sqrt(0.5 + 0.5 * vn) - vn) * np.sqrt(ALPHA)


# ---- closed forms for pure absorbers seen face-on --------------------------------------------------------------------------
def absorber_expectation(medium, hz, ior, max_depth, L_down, L_up=None):
    """E of a pixel of the +z face of a box of half-depth hz, seen face-on, for a medium with sigma_s = 0.

    Every ray meets the faces at normal incidence.  A boundary interaction reflects with probability F (the Fresnel
    reflectance at normal incidence, the same from either side) and transmits with probability 1 - F, with weight 1 either
    way, and each crossing of the box (length s, `segment`) is weighted T = exp(-sigma_t s).  A path that enters and leaves
    after j crossings (j - 1 internal reflections) has probability (1 - F)^2 F^(j - 1), weight T^j, and leaves downwards for
    odd j, upwards for even j; a path reflected at the first hit leaves upwards with probability F.  The environment is
    reached at the bounce after the last boundary interaction: interactions are bounces 0 .. j, so the miss is at depth j + 1
    (depth 1 for the first reflection), and it is only taken while depth < maxDepth: j <= maxDepth - 2.  Russian roulette from
    depth 3 divides by its continuation probability and so leaves the expectation unchanged.  So

        E = F L_up [maxDepth >= 2] + sum_{j=1}^{maxDepth-2} (1 - F)^2 F^(j-1) T^j L_(j odd ? down : up).

    With ior 1, F = 0 and E = L_down T for maxDepth >= 3."""
    L_up = L_down if L_up is None else L_up
    L_down, L_up = np.asarray(L_down, np.float64), np.asarray(L_up, np.float64)
    F = float(fresnel(ior, fcos(1.0)))
    T = np.exp(-medium.walk[0] * segment(hz)) if medium.present else np.ones(3)
    E = F * L_up if max_depth >= 2 else np.zeros(3)
    for j in range(1, max_depth - 1):
        E = E + (1 - F) ** 2 * F ** (j - 1) * T ** j * (L_down if j % 2 else L_up)
    return E


# ---- Monte Carlo of the estimator for scattering media ---------------------------------------------------------------------
def _frame(w):
    """two unit vectors orthogonal to the unit vectors w [n, 3]"""
    a = np.where(np.abs(w[:, :1]) < 0.9, np.array([[1.0, 0, 0]]), np.array([[0, 1.0, 0]]))
    t = np.cross(w, a)
    t /= np.linalg.norm(t, axis=1, keepdims=True)
    return t, np.cross(w, t)


def _exit(p, d, h):
    """distance along d from p (inside the box of half extents h) to the boundary, and the outward normal there"""
    with np.errstate(divide="ignore", invalid="ignore"):
        t = np.where(d > 0, (h - p) / d, np.where(d < 0, (-h - p) / d, np.inf))
    ax = np.argmin(t, 1)
    n = np.zeros_like(p)
    n[np.arange(len(p)), ax] = np.sign(d[np.arange(len(p)), ax])
    return np.maximum(t[np.arange(len(p)), ax], 0.0), n


class Lighting:
    """The lights and the environment as sampleLights sees them: `env` an estref.Env (or None), its rotation and
    intensity, and the b200pt_light records."""

    def __init__(self, env=None, rotation=0.0, intensity=1.0, lights=()):
        self.env, self.rot, self.inten, self.lights = env, rotation, intensity, list(lights)
        self.env_on = env is not None and intensity > 0
        self.lw, self.ew = estref.technique_probabilities(len(self.lights), self.env_on)
        if env is not None:
            self.cdf = np.cumsum(env.texel_prob().reshape(-1))

    def lookup(self, d_world):
        """rgb * intensity and alpha of the environment in world directions"""
        look = self.env.lookup(estref.rotate_y(d_world, -self.rot))
        return look[:, :3] * self.inten, look[:, 3]

    def sample_env(self, rng, n):
        """environmentSample: a texel with the realised alias-table probabilities, uniform in (phi, cos theta) inside it"""
        e = self.env
        i = np.minimum(np.searchsorted(self.cdf, rng.random(n) * self.cdf[-1], side="right"), e.w * e.h - 1)
        row, col = i // e.w, i % e.w
        phi = (col + rng.random(n)) / e.w * estref.TWO_PI - np.pi
        x = rng.random(n)
        ct = e.cos_edges[row] * (1 - x) + e.cos_edges[row + 1] * x
        return estref.rotate_y(estref.phi_cos_to_dir(phi, ct), self.rot)


def nee(light, med, h, ior, p, wi, rng, rte=()):
    """volumeScatterNEE at the points p [n, 3] with incoming directions wi: the value per unit throughput [n, 3]"""
    n = len(p)
    out = np.zeros((n, 3))
    if light.lw == 0 and light.ew == 0:
        return out
    use_light = rng.random(n) < light.lw
    dirs = np.zeros((n, 3))
    rad = np.zeros((n, 3))
    pdf = np.zeros(n)
    dist = np.full(n, np.inf)
    dirac = np.zeros(n, bool)
    idx = np.nonzero(use_light)[0]
    if len(idx):
        nl = len(light.lights)
        j = np.minimum((rng.random(len(idx)) * nl).astype(int), nl - 1)
        for k, L in enumerate(light.lights):
            sel = idx[j == k]
            if not len(sel):
                continue
            assert L.type == 3 and L.angularSizeOrInvRange == 0, "point and sphere lights without range only"
            l2s = p[sel] - np.array(L.position[:], np.float64)
            dist[sel] = np.linalg.norm(l2s, axis=1)
            wdir = -l2s / dist[sel, None]
            color = np.array(L.color[:], np.float64)
            if L.radius == 0:
                dirs[sel], dirac[sel] = wdir, True
                rad[sel] = (L.intensity / dist[sel] ** 2)[:, None] * color / ((1.0 / nl) * light.lw)
                continue
            halfang = np.arctan(np.minimum(L.radius / dist[sel], 1.0))
            cmax = np.cos(halfang)
            ct = 1.0 - rng.random(len(sel)) * (1.0 - cmax)
            ph = estref.TWO_PI * rng.random(len(sel))
            t, b = _frame(wdir)
            st = np.sqrt(np.maximum(0.0, 1.0 - ct * ct))
            dirs[sel] = (t * np.cos(ph)[:, None] + b * np.sin(ph)[:, None]) * st[:, None] + wdir * ct[:, None]
            rad[sel] = (L.intensity / L.radius ** 2 * halfang ** 2)[:, None] * color / ((1.0 / nl) * light.lw)
            pdf[sel] = 1.0 / (estref.TWO_PI * (1.0 - cmax)) / nl
        lit = idx[~dirac[idx]]
        env_pdf = light.lookup(dirs[lit])[1] if light.env_on and len(lit) else 0.0
        psum = light.lw * pdf[lit] + light.ew * env_pdf
        rad[lit] *= (light.lw * pdf[lit] / psum)[:, None]
        pdf[lit] = psum
    idx = np.nonzero(~use_light)[0]
    if len(idx) and light.env_on:
        d = light.sample_env(rng, len(idx))
        rgb, alpha = light.lookup(d)
        dirs[idx], rad[idx], pdf[idx] = d, rgb / (alpha * light.ew)[:, None], light.ew * alpha
    cos = np.sum(wi * dirs, 1)
    phase = hg_pdf(cos, med.g)
    with np.errstate(divide="ignore", invalid="ignore"):
        w = np.where(pdf > 0, pdf / (pdf + phase), 0.0)
    if "dirac" in rte:
        w = np.where(dirac, 1.0, w)
    ok = (pdf > 0) | (dirac & ("dirac" in rte))
    t, nrm = _exit(p, dirs, h)
    t = np.minimum(t, dist)
    sig_t, _ = med.full
    shadow = (1.0 - R.schlick(((ior - 1) / (ior + 1)) ** 2, np.abs(np.sum(dirs * nrm, 1))))[:, None] * np.exp(-sig_t[None] * t[:, None])
    if med.shadow_scatters and "shadow" not in rte:
        shadow *= np.exp(-sig_t.max() * t)[:, None]
    shadow = np.where(shadow.max(1, keepdims=True) <= 0.01, 0.0, shadow)
    return np.where(ok[:, None], rad * (w * phase)[:, None] * shadow, 0.0)


def _boundary(d, nrm_out, inside, ior, rng):
    """the smooth dielectric at a face with outward normal nrm_out: new direction and new inside flag"""
    N = np.where((np.sum(-d * nrm_out, 1) > 0)[:, None], nrm_out, -nrm_out)
    k = -d
    vn = np.clip(np.sum(k * N, 1), 0.0, 1.0)
    ior1 = np.where(inside, ior, 1.0)
    ior2 = np.where(inside, 1.0, ior)
    F = fresnel(ior2 / ior1, fcos(vn))
    refl = rng.random(len(d)) < F
    b = ior1 / ior2
    s2 = b * b * (1.0 - vn * vn)
    tir = s2 >= 1.0
    tdir = -b[:, None] * k + N * (b * vn - np.sqrt(np.maximum(0.0, 1.0 - s2)))[:, None]
    rdir = 2.0 * vn[:, None] * N - k
    mirror = refl | tir
    out = np.where(mirror[:, None], rdir, tdir)
    out /= np.linalg.norm(out, axis=1, keepdims=True)
    return out, np.where(mirror, inside, ~inside)


def monte_carlo(med, light, half_ext, ior, max_depth, view, n, seed=1, rte=(), chunk=1 << 17):
    """E of one sample through the +z face of the box with half extents `half_ext`, the entry point uniform over
    [-view, view]^2, as a float64 Monte Carlo of the estimator (module docstring): (E [3], standard error [3]).  `rte`
    may hold "shadow" (one exp(-sigma_t d) on shadow rays), "dirac" (Dirac lights lit through the medium with weight 1) and
    "null" (weighted delta tracking: a collision is a real scatter or a null collision that keeps the direction, and a
    segment that reaches the boundary has weight 1)."""
    rng = np.random.default_rng(seed)
    h = np.asarray(half_ext, np.float64)
    sig_t, sig_s = med.walk
    m = sig_t.max()
    g = med.g
    sums, sq = np.zeros(3), np.zeros(3)
    done = 0
    while done < n:
        c = min(chunk, n - done)
        p = np.stack([rng.uniform(-view, view, c), rng.uniform(-view, view, c), np.full(c, h[2])], 1)
        d = np.tile([0.0, 0.0, -1.0], (c, 1))
        thr = np.ones((c, 3))
        rad = np.zeros((c, 3))
        inside = np.zeros(c, bool)
        depth = np.zeros(c, int)
        nscat = np.zeros(c, int)
        alive = np.ones(c, bool)
        first = np.ones(c, bool)
        while alive.any():
            a = np.nonzero(alive)[0]
            # a ray outside the box after a bounce leaves the scene: the environment, while depth < maxDepth
            out = a[~inside[a] & ~first[a]]
            if len(out):
                ok = out[depth[out] < max_depth]
                if len(ok) and light.env_on:
                    rad[ok] += thr[ok] * light.lookup(d[ok])[0]
                alive[out] = False
            a = np.nonzero(alive)[0]
            if not len(a):
                break
            # distance to the boundary; for the camera ray the +z face at distance 0
            t, nrm = _exit(p[a], d[a], h)
            t = np.where(first[a], 0.0, t)
            nrm[first[a]] = (0.0, 0.0, 1.0)
            scat = np.zeros(len(a), bool)
            med_on = inside[a] & med.present
            if med.scatters:
                s = -np.log(np.maximum(rng.random(len(a)), 1e-10)) / m
                scat = med_on & (s < t)
                pas = med_on & ~scat
                if "null" in rte:
                    ps = min(sig_s.sum() / (sig_s.sum() + (m - sig_t).sum()), 1.0 - 1e-12)
                    real = rng.random(len(a)) < ps
                    nul = scat & ~real
                    i = a[nul]
                    thr[i] *= (m - sig_t) / (m * (1 - ps))
                    p[i] += d[i] * s[nul, None]
                    scat = scat & real
                    # a null collision continues along the same direction: next iteration
                    pas_w = np.ones(3)
                else:
                    pas_w = None
                i = a[pas]
                if pas_w is None:
                    thr[i] *= np.exp((m - sig_t)[None] * t[pas, None])
                i = a[scat]
                if len(i):
                    wi = d[i].copy()
                    thr[i] *= 1.0 - (sig_t - sig_s) / m if "null" not in rte else sig_s / (m * ps)
                    p[i] += wi * s[scat, None]
                    rad[i] += thr[i] * nee(light, med, h, ior, p[i], wi, rng, rte)
                    ct = hg_cos(rng.random(len(i)), g)
                    ph = estref.TWO_PI * rng.random(len(i))
                    tt, bb = _frame(wi)
                    st = np.sqrt(np.maximum(0.0, 1.0 - ct * ct))
                    d[i] = (tt * np.cos(ph)[:, None] + bb * np.sin(ph)[:, None]) * st[:, None] + wi * ct[:, None]
                    d[i] /= np.linalg.norm(d[i], axis=1, keepdims=True)
                    nscat[i] += 1
                    rr = i[nscat[i] >= 64]
                    if len(rr):
                        q = np.minimum(thr[rr].max(1) + 0.001, 0.95)
                        live = rng.random(len(rr)) < q
                        alive[rr[~live]] = False
                        thr[rr[live]] /= q[live, None]
                if "null" in rte:
                    nul_mask = np.zeros(len(a), bool)
                    nul_mask[nul] = True
                    scat = scat | nul_mask
            elif med.present:
                i = a[med_on]
                thr[i] *= np.exp(-sig_t[None] * t[med_on, None])
            # the boundary bounce
            b = a[~scat]
            if not len(b):
                continue
            bt = t[~scat]
            p[b] += d[b] * bt[:, None]
            d[b], inside[b] = _boundary(d[b], nrm[~scat], inside[b], ior, rng)
            first[b] = False
            rr = b[depth[b] >= 3]
            if len(rr):
                q = np.minimum(thr[rr].max(1) + 0.001, 0.95)
                live = rng.random(len(rr)) < q
                alive[rr[~live]] = False
                thr[rr[live]] /= q[live, None]
            depth[b] += 1
            stop = b[(depth[b] >= max_depth) & alive[b]]
            alive[stop] = False
        sums += rad.sum(0)
        sq += (rad * rad).sum(0)
        done += c
    mean = sums / n
    var = sq / n - mean * mean
    return mean, np.sqrt(np.maximum(var, 0.0) / n)
