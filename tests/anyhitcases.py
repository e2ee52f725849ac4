"""Scenes, rays and checks shared by test_anyhit_expectation.py (the CPU oracle) and test_gpu_anyhit_expectation.py (the
device): the any-hit loops of trace_closest / trace_shadow against the float64 model of tests/anyhitref.py.

A case is a scene, closest-hit rays and shadow rays with a seed each.  Two kinds of check run on what an implementation
returns (hits or transmission, and the seeds it handed back):
  * per ray, on the rays the model does not flag: the replay of the ray's draws in t order predicts the hit (render node and
    triangle; inside a group of crossings at bit-identical t, any member, at the replayed position), t within 1e-5, the
    barycentrics within 1e-4, the shadow transmission within 1e-5 (0 exactly), and the number of draws exactly -- read by
    stepping the generator from the seed in to the seed out;
  * over all unflagged rays, without any order: a chi-square of where the rays stop (per layer, the opaque hit, a miss)
    against the summed probabilities p_i prod_{j<i} (1 - p_j), and the mean number of draws and the mean transmission per
    channel within 4.5 sigma of their expectations.
A fraction of each case's seeds is chosen so that the first draw equals the first candidate's opacity exactly: the closest
test accepts there (rand() <= opacity) and the shadow test does not (rand() < opacity).
"""
import functools
import math

import numpy as np
from scipy import stats

import anyhitref as ah
from vk_gltf_renderer_b200 import synth
from vk_gltf_renderer_b200.scene import Camera, Scene

VEIL_COUNTS = (1, 3, 4, 5, 12, 13, 28, 29, 45)   # around kCand = 4, kCand (1 + R) at R = 2, one and two walks of 16 beyond
MAX_FLAGGED = 0.005
N_SIGMA = 4.5
P_MIN = 1e-4
STAT_RAYS = 1 << 18


def _grid(a):
    """an alpha on the draw grid (k 2^-23), so that a chosen seed can land a draw exactly on it"""
    return float(np.float32(round(a * 2.0 ** 23) * ah.GRID))


def _quad(scn, x0, x1, y0, y1, z=0.0, uv=True, colors=None):
    pos = [[x0, y0, z], [x1, y0, z], [x1, y1, z], [x0, y1, z]]
    return scn.add_primitive(pos, [[0, 1, 2], [0, 2, 3]], normals=[[0, 0, 1]] * 4,
                             uv0=[[0, 0], [1, 0], [1, 1], [0, 1]] if uv else None, colors=colors)


def _blend(scn, alpha, double_sided=1, **kw):
    return scn.add_material(pbrBaseColorFactor=[1, 1, 1, alpha], pbrMetallicFactor=0.0, pbrRoughnessFactor=0.8, alphaMode=2,
                            doubleSided=double_sided, **kw)


def _wall(scn, z, x=(-4.0, 4.0)):
    m = scn.add_material(pbrBaseColorFactor=[0.5, 0.5, 0.5, 1], pbrMetallicFactor=0.0, doubleSided=1)
    scn.add_node(_quad(scn, x[0], x[1], -4.0, 4.0, z), m)


def _camera(scn):
    cam = Camera()
    cam.eye = np.array([0.0, 0.0, 3.0], np.float32)
    cam.center = np.array([0.0, 0.0, 0.0], np.float32)
    cam.yfov = math.radians(45.0)
    cam.znear, cam.zfar = 0.05, 100.0
    scn.camera = cam
    return scn


def veils(n, double_sided=True, spacing=0.05, seed=7):
    """n parallel BLEND quads of constant alpha 0.05-0.15 (the second one 0) at z = -spacing i, a small alpha-1 quad half-way
    down the stack and an opaque wall behind it"""
    rng = np.random.default_rng(seed + n)
    scn = Scene()
    prim = _quad(scn, -1.0, 1.0, -1.0, 1.0)
    for i in range(n):
        a = 0.0 if (i == 1 and n >= 3) else _grid(rng.uniform(0.05, 0.15))
        scn.add_node(prim, _blend(scn, a, 1 if double_sided else 0), np.diag([1.0, 1.0, 1.0, 1.0]) + _tz(-spacing * i))
    cap = _quad(scn, 0.2, 0.8, 0.2, 0.8, -spacing * (n // 2) - spacing / 2)
    scn.add_node(cap, _blend(scn, 1.0, 1 if double_sided else 0))
    _wall(scn, -spacing * n - 0.2)
    return _camera(scn)


def _tz(z):
    m = np.zeros((4, 4))
    m[2, 3] = z
    return m


def ties(copies=20):
    """`copies` render nodes of one quad with identity matrices (bit-identical t, equal opacity), three layers behind"""
    scn = Scene()
    prim = _quad(scn, -1.0, 1.0, -1.0, 1.0)
    m = _blend(scn, _grid(0.1))
    for _ in range(copies):
        scn.add_node(prim, m)
    for k, a in enumerate((0.3, 0.5, 0.7)):
        scn.add_node(_quad(scn, -1.0, 1.0, -1.0, 1.0, -0.3 * (k + 1)), _blend(scn, _grid(a)))
    _wall(scn, -1.2)
    return _camera(scn)


def mirrored(fillers=10):
    """three BLEND layers whose alpha runs along texture u -- one under a mirroring node, one under a rotated and scaled node,
    one with a different vertex alpha at each corner -- in front of `fillers` constant layers and again behind them"""
    scn = Scene()
    ramp = np.full((1, 64, 4), 255, np.uint8)
    ramp[0, :, 3] = np.linspace(0, 255, 64).astype(np.uint8)
    ti = scn.add_texture_info(scn.add_texture(ramp, srgb=False, wrapS=33071, wrapT=33071, magFilter=9729, minFilter=9987))
    grad = _blend(scn, 1.0, pbrBaseColorTexture=ti)
    plain = _quad(scn, -1.0, 1.0, -1.0, 1.0)
    col = (np.array([40, 120, 200, 255], np.uint32) << np.uint32(24)) | np.uint32(0x00FFFFFF)
    tinted = _quad(scn, -1.0, 1.0, -1.0, 1.0, colors=col)
    filler = _blend(scn, _grid(0.05))
    c, s = math.cos(0.5), math.sin(0.5)

    def trio(z):
        scn.add_node(plain, grad, np.diag([-1.0, 1.0, 1.0, 1.0]) + _tz(z))
        rot = np.array([[c * 1.3, -s * 0.8, 0, 0], [s * 1.3, c * 0.8, 0, 0], [0, 0, 1, z - 0.04], [0, 0, 0, 1]])
        scn.add_node(plain, grad, rot)
        scn.add_node(tinted, grad, np.eye(4) + _tz(z - 0.08))
    trio(0.0)
    for k in range(fillers):
        scn.add_node(plain, filler, np.eye(4) + _tz(-0.15 - 0.05 * k))
    trio(-0.2 - 0.05 * fillers)
    _wall(scn, -0.5 - 0.05 * fillers)
    return _camera(scn)


def occluded():
    """five BLEND layers, an opaque wall covering x < 0.3, six BLEND layers behind it, a back wall"""
    scn = Scene()
    prim = _quad(scn, -1.0, 1.0, -1.0, 1.0)
    rng = np.random.default_rng(3)
    for k in range(5):
        scn.add_node(prim, _blend(scn, _grid(rng.uniform(0.05, 0.15))), np.eye(4) + _tz(-0.1 * k))
    _wall(scn, -0.55, x=(-4.0, 0.3))
    for k in range(6):
        scn.add_node(prim, _blend(scn, _grid(rng.uniform(0.05, 0.15))), np.eye(4) + _tz(-0.7 - 0.1 * k))
    _wall(scn, -1.5)
    return _camera(scn)


def tinted():
    """synth_layers(tinted=True) (14 transmissive sheets) behind a closed BLEND slab of thickness > 0 with an attenuation
    colour"""
    scn = synth.synth_layers(tinted=True)
    m = scn.add_material(pbrBaseColorFactor=[0.95, 0.9, 0.85, 0.6], pbrRoughnessFactor=0.2, pbrMetallicFactor=0.0, alphaMode=2,
                         transmissionFactor=0.8, thicknessFactor=0.5, attenuationColor=[0.6, 0.8, 0.9], attenuationDistance=0.7, ior=1.4)
    lo, hi = np.array([-1.2, 0.3, 0.3]), np.array([1.3, 1.9, 0.7])
    c = np.array([[x, y, z] for z in (lo[2], hi[2]) for y in (lo[1], hi[1]) for x in (lo[0], hi[0])])
    faces = [[0, 2, 3], [0, 3, 1], [4, 5, 7], [4, 7, 6], [0, 1, 5], [0, 5, 4], [2, 6, 7], [2, 7, 3], [0, 4, 6], [0, 6, 2],
             [1, 3, 7], [1, 7, 5]]
    scn.add_node(scn.add_primitive(c, faces), m)
    return scn


SCENES = {
    "ties": ties,
    "textured": synth.sampler_layers,
    "mirrored": mirrored,
    "mask": synth.synth_layers,
    "tinted": tinted,
    "occluded": occluded,
}


def scene_of(name):
    if name.startswith("veils"):
        _, n, sides = name.split("-")
        return veils(int(n), sides == "2s")
    return SCENES[name]()


# ---- rays ------------------------------------------------------------------------------------------------------------------
def _rays(o, tgt, tmax=1e32):
    d = tgt - o
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    r = np.zeros((len(o), 8), np.float32)
    r[:, 0:3], r[:, 4:7], r[:, 7] = o, d, tmax
    return r


def stack_rays(n, z_front, z_back, half, rng, between=0.4, back=0.15):
    """rays through a stack of layers in z_back < z < z_front, |x|, |y| < half: from outside in front, from between the layers
    towards the back (a fraction with tmin > 0) and from between the layers out of the front (back faces)"""
    kind = rng.random(n)
    o = np.stack([rng.uniform(-half, half, n), rng.uniform(-half, half, n), rng.uniform(z_front + 0.3, z_front + 2.0, n)], 1)
    inner = kind < between
    o[inner, 2] = rng.uniform(z_back, z_front, inner.sum())
    o[inner, :2] *= 0.7
    tgt = np.stack([rng.uniform(-half, half, n), rng.uniform(-half, half, n), np.full(n, z_back - 1.0)], 1)
    out = kind < back
    tgt[out, 2] = z_front + 2.0
    r = _rays(o, tgt)
    tmin = (rng.random(n) < 0.3) * rng.uniform(0.0, 0.4, n)
    r[:, 3] = tmin.astype(np.float32)
    return r


def shadow_cut(rays, z_cut, rng):
    """shadow rays: tmin 0 (the renderer's ray-level API starts every shadow ray at its origin, so the cases give them no tmin
    of their own), tmax at a random depth between the origin and the plane z = z_cut (some beyond everything)"""
    r = rays.copy()
    r[:, 3] = 0.0
    dz = r[:, 6].astype(np.float64)
    with np.errstate(divide="ignore"):
        t_cut = np.where(dz < -1e-3, (z_cut - r[:, 2]) / dz, 4.0)
    r[:, 7] = (t_cut * rng.uniform(0.05, 1.0, len(r))).astype(np.float32)
    far = rng.random(len(r)) < 0.1
    r[far, 7] = 1e32
    return r


def rays_of(name, n, seed=5):
    rng = np.random.default_rng(seed)
    if name.startswith("veils"):
        k = int(name.split("-")[1])
        z_back = -0.05 * k - 0.2
        rays = stack_rays(n, 0.02, z_back + 0.15, 1.0, rng)
        return rays, shadow_cut(rays, z_back, rng)
    if name == "ties":
        rays = stack_rays(n, 0.02, -0.95, 1.0, rng, between=0.0, back=0.0)
        return rays, shadow_cut(rays, -1.2, rng)
    if name == "mirrored":
        rays = stack_rays(n, 0.02, -0.95, 0.8, rng)
        return rays, shadow_cut(rays, -1.0, rng)
    if name == "occluded":
        rays = stack_rays(n, 0.02, -1.3, 1.0, rng)
        return rays, shadow_cut(rays, -1.5, rng)
    # the synth_layers family: 14 layers at z = 0 .. -1.95, x in [-1.5, 1.6], y in [0.1, 2.1], a floor at y = 0
    o = np.stack([rng.uniform(-1.4, 1.4, n), rng.uniform(0.2, 2.0, n), rng.uniform(0.5, 3.0, n)], 1)
    inner = rng.random(n) < 0.25
    o[inner, 2] = rng.uniform(-1.9, 0.0, inner.sum())
    tgt = np.stack([rng.uniform(-1.4, 1.4, n), rng.uniform(0.2, 2.0, n), np.full(n, -2.4)], 1)
    rays = _rays(o, tgt)
    sh = rays.copy()
    sh[:, 7] = (np.linalg.norm(tgt - o, axis=1) * rng.uniform(0.3, 1.0, n)).astype(np.float32)
    return rays, sh


def plain_seeds(n, salt):
    return ((np.arange(n, dtype=np.uint64) * np.uint64(2654435761) + np.uint64(salt)) % np.uint64(1 << 32)).astype(np.uint32)


class Case:
    """a scene, its rays and seeds, and the model's predictions (computed once)"""

    def __init__(self, name, n):
        self.name = name
        self.scn = scene_of(name)
        self.rays, self.rays_s = rays_of(name, n)
        self.model = ah.SceneModel(self.scn)
        self.closest = None if name == "tinted" else self._closest()
        self.shadow = self._shadow()

    def _edge_seeds(self, cr, a, cand):
        """plain seeds, and for every eighth ray with a candidate one whose first draw is that candidate's opacity"""
        seeds = plain_seeds(len(cr["n"]), 777)
        has = cand.any(1) & (np.arange(len(seeds)) % 8 == 0)
        first = np.argmax(cand, 1)
        k = np.round(a[np.arange(len(seeds)), first] * 2.0 ** 23)
        on_grid = has & (k * ah.GRID == a[np.arange(len(seeds)), first]) & (k < 2 ** 23)
        for r in np.nonzero(on_grid)[0]:
            seeds[r] = ah.seed_for_first_draw(int(k[r]))
        return seeds, on_grid

    def _closest(self):
        M = self.model
        cr = M.crossings(self.rays, shadow=False)
        a, err, opq = M.opacity(cr)
        cand, _ = ah._candidates(cr, opq)
        seeds, edge = self._edge_seeds(cr, a, cand)
        hit, used, flag = ah.replay_closest(cr, a, err, opq, seeds)
        stop, p_opq, p_miss, e_d, var_d = ah.closest_expectation(cr, a, opq)
        layer = M.layer_of(cr)
        tri = np.where(cr["valid"], M.tri[np.maximum(cr["j"], 0)], -2)
        # only what the checks read, in narrow types: t, u, v in float32 keep every distinct t apart (near-ties are flagged)
        return dict(t=cr["t"].astype(np.float32), u=cr["u"].astype(np.float32), v=cr["v"].astype(np.float32),
                    layer=layer.astype(np.int32), tri=tri.astype(np.int32), seeds=seeds, edge=edge, hit=hit, used=used,
                    flag=flag | cr["flag"], stop=stop.astype(np.float32), p_opq=p_opq, p_miss=p_miss, e_d=e_d, var_d=var_d,
                    group=_tie_groups(cr["t"], layer))

    def _shadow(self):
        M = self.model
        cr = M.crossings(self.rays_s, shadow=True)
        a, err, opq = M.opacity(cr)
        c, thick, absorb = M.transmission(cr, self.rays_s[:, 4:7])
        cand = cr["valid"] & ~opq & ~(cr["valid"] & opq).any(1)[:, None]
        seeds, edge = self._edge_seeds(cr, a, cand)
        T, used, flag = ah.replay_shadow(cr, a, err, opq, c, thick, absorb, seeds)
        ET, ET2, ED, ED2 = ah.shadow_expectation(cr, a, opq, c, thick, absorb)
        return dict(seeds=seeds, edge=edge, T=T, used=used, flag=flag | cr["flag"], ET=ET, var_T=ET2 - ET * ET, e_d=ED, var_d=ED2 - ED * ED)


def _tie_groups(t, layer):
    """render node -> the smallest render node it is ever crossed at a bit-identical t with (union of such pairs): the
    members of a tie group come in an order the reference leaves open, so the stop distribution counts each group once"""
    parent = {}

    def find(x):
        while parent.setdefault(x, x) != x:
            x = parent[x]
        return x
    same = (t[:, 1:] == t[:, :-1]) & np.isfinite(t[:, 1:])
    pairs = np.unique(np.stack([layer[:, 1:][same], layer[:, :-1][same]], 1), axis=0)
    for a, b in pairs:
        ra, rb = find(int(a)), find(int(b))
        parent[max(ra, rb)] = min(ra, rb)
    return {k: find(k) for k in list(parent)}


@functools.lru_cache(maxsize=None)
def case(name, n=STAT_RAYS):
    return Case(name, n)


# ---- checks ------------------------------------------------------------------------------------------------------------------
def _mean_check(got, expect, var, label, report):
    n = len(got)
    mean, E = float(np.mean(got)), float(np.mean(expect))
    sigma = math.sqrt(float(np.sum(np.maximum(var, 0.0)))) / n
    report.append(f"{label}: mean {mean:.6g} E {E:.6g} sigma {sigma:.3g}")
    assert abs(mean - E) <= N_SIGMA * sigma + 1e-9 * max(abs(E), 1.0), report[-1]


def _chi_square(observed, expected, label, report):
    order = np.argsort(expected)
    pooled_o, pooled_e, acc_o, acc_e = [], [], 0.0, 0.0
    for i in order:
        acc_o += observed[i]
        acc_e += expected[i]
        if acc_e >= 5.0:
            pooled_o.append(acc_o), pooled_e.append(acc_e)
            acc_o = acc_e = 0.0
    if acc_e > 0 or acc_o > 0:
        if pooled_e:
            pooled_o[-1] += acc_o
            pooled_e[-1] += acc_e
        else:
            pooled_o.append(acc_o), pooled_e.append(acc_e)
    o, e = np.array(pooled_o), np.array(pooled_e)
    chi2 = float(np.sum((o - e) ** 2 / np.maximum(e, 1e-300)))
    p = float(stats.chi2.sf(chi2, max(len(o) - 1, 1))) if len(o) > 1 else 1.0
    report.append(f"{label}: {len(o)} categories, chi2 {chi2:.2f}, p {p:.3g}")
    assert len(o) <= 1 or p >= P_MIN, report[-1]
    if len(o) == 1:
        assert o[0] == e[0] or abs(o[0] - e[0]) < 1e-6 * e[0] + 1e-9, report[-1]


def check_closest(c, hits, seeds_out, report, count_draws=True, rows=None):
    """hits float32 [n, 6] (t, render node, render primitive, triangle, u, v) and the seeds returned, for the case's first n
    rays (or the rays `rows`)"""
    m = c.closest
    rows = np.arange(len(hits)) if rows is None else rows
    ids = hits.view(np.int32)
    flag = m["flag"][rows]
    report.append(f"{c.name} closest: {len(rows)} rays, {flag.mean():.3%} flagged")
    assert flag.mean() < MAX_FLAGGED, report[-1]
    ok = ~flag
    r = rows[ok]
    h = m["hit"][r]
    got_node, got_tri = ids[ok, 1], ids[ok, 3]
    miss = h < 0
    bad = np.zeros(len(r), bool)
    bad |= miss & (got_node != -1)
    hh = np.maximum(h, 0)
    t_pred = m["t"][r, hh]
    same_t = m["t"][r] == t_pred[:, None]
    member = (same_t & (m["layer"][r] == got_node[:, None]) & (m["tri"][r] == got_tri[:, None])).any(1)
    bad |= ~miss & ~member
    bad |= ~miss & (np.abs(hits[ok, 0] - t_pred) > 1e-5 * np.maximum(t_pred, 1e-3))
    bad |= ~miss & ((np.abs(hits[ok, 4] - m["u"][r, hh]) > 1e-4) | (np.abs(hits[ok, 5] - m["v"][r, hh]) > 1e-4))
    if count_draws:
        used = ah.steps_between(m["seeds"][r], seeds_out[ok], max_steps=int(m["used"].max()) + 4)
        bad |= used != m["used"][r]
    report.append(f"{c.name} closest: {int(bad.sum())} of {len(r)} unflagged rays differ from the replay")
    if bad.any():
        i = np.nonzero(bad)[0][:5]
        report.append(f"  first rays {r[i].tolist()}: predicted crossing {h[i].tolist()} used {m['used'][r[i]].tolist()}, "
                      f"got node {got_node[i].tolist()} tri {got_tri[i].tolist()} t {hits[ok, 0][i].tolist()}")
    assert not bad.any(), "\n".join(report[-2:])


def check_closest_distribution(c, hits, seeds_out, report, count_draws=True, rows=None):
    """the stop distribution and the mean number of draws over the unflagged rays of `rows` (default: the case's first
    len(hits)) whose seeds were not chosen; one category per layer -- a tie group counts as one layer --, the opaque hit and
    the miss"""
    m = c.closest
    rows = np.arange(len(hits)) if rows is None else rows
    ok = ~m["flag"][rows] & ~m["edge"][rows]     # the chosen first draws are not random
    r = rows[ok]
    if not len(r):
        return
    got_node = hits.view(np.int32)[ok, 1]
    group = lambda x: np.vectorize(lambda k: m["group"].get(int(k), int(k)), otypes=[np.int64])(x) if x.size else x
    layer = group(m["layer"][r])
    stop = m["stop"][r].astype(np.float64)
    opaque_nodes = sorted({int(c.model.node[k]) for k in np.nonzero(c.model.opaque)[0]})
    got = group(got_node)
    cats = sorted((set(np.unique(layer[layer >= 0]).tolist()) | set(np.unique(got[got >= 0]).tolist())) - set(opaque_nodes))
    expected = [float(stop[layer == k].sum()) for k in cats] + [float(m["p_opq"][r].sum()), float(m["p_miss"][r].sum())]
    observed = [float((got == k).sum()) for k in cats] + [float(np.isin(got_node, opaque_nodes).sum()), float((got_node == -1).sum())]
    _chi_square(np.array(observed), np.array(expected), f"{c.name} closest stops", report)
    if count_draws:
        used = ah.steps_between(m["seeds"][r], seeds_out[ok], max_steps=int(m["used"].max()) + 4)
        _mean_check(used, m["e_d"][r], m["var_d"][r], f"{c.name} closest draws", report)


def check_shadow(c, T, seeds_out, report, count_draws=True, rows=None):
    m = c.shadow
    rows = np.arange(len(T)) if rows is None else rows
    flag = m["flag"][rows]
    report.append(f"{c.name} shadow: {len(rows)} rays, {flag.mean():.3%} flagged")
    assert flag.mean() < MAX_FLAGGED, report[-1]
    ok = ~flag
    r = rows[ok]
    pred, got = m["T"][r], T[ok].astype(np.float64)
    bad = ((pred == 0) != (got == 0)).any(1)
    bad |= (np.abs(got - pred) > 1e-5 * np.maximum(np.abs(pred), 1e-30)).any(1)
    if count_draws:
        used = ah.steps_between(m["seeds"][r], seeds_out[ok], max_steps=int(m["used"].max()) + 4)
        bad |= used != m["used"][r]
    report.append(f"{c.name} shadow: {int(bad.sum())} of {len(r)} unflagged rays differ from the replay")
    if bad.any():
        i = np.nonzero(bad)[0][:5]
        report.append(f"  first rays {r[i].tolist()}: predicted {pred[i].tolist()} used {m['used'][r[i]].tolist()}, got {got[i].tolist()}")
    assert not bad.any(), "\n".join(report[-2:])


def check_shadow_distribution(c, T, seeds_out, report, count_draws=True, rows=None):
    m = c.shadow
    rows = np.arange(len(T)) if rows is None else rows
    ok = ~m["flag"][rows] & ~m["edge"][rows]
    r = rows[ok]
    if not len(r):
        return
    for ch in range(3):
        _mean_check(T[ok, ch].astype(np.float64), m["ET"][r, ch], m["var_T"][r, ch], f"{c.name} shadow T[{ch}]", report)
    if count_draws:
        used = ah.steps_between(m["seeds"][r], seeds_out[ok], max_steps=int(m["used"].max()) + 4)
        _mean_check(used, m["e_d"][r], m["var_d"][r], f"{c.name} shadow draws", report)


# ---- the frame path: k_trace / k_shadow -> k_alpha inside a rendered frame --------------------------------------------------
EMISSIVE_VEIL_COUNTS = (1, 5, 13, 29)
SHADOW_VEIL_COUNTS = (1, 5, 13)
SHADOW_LIGHT_DIR = (1.0, -0.6, 0.3)       # direction of travel: the light stands to the side, away from the camera's view


def _black(scn, alpha, emission=(0.0, 0.0, 0.0), double_sided=1):
    """a BLEND layer that neither reflects nor transmits (base colour 0, metallic 0, specularFactor 0): all it can do to a
    path is end it, and add its emission"""
    return scn.add_material(pbrBaseColorFactor=[0, 0, 0, alpha], pbrMetallicFactor=0.0, pbrRoughnessFactor=1.0, specularFactor=0.0,
                            emissiveFactor=list(emission), alphaMode=2, doubleSided=double_sided)


def emissive_veils(n, L, seed=21):
    """n black BLEND layers with distinct emission e_i filling the view of an orthographic camera, in front of a constant
    environment L.  Every pixel has the same expectation sum_i e_i p_i prod_{j<i} (1 - p_j) + L prod_j (1 - p_j), p on the
    closest-hit grid.  Returns (scene, E [3])."""
    rng = np.random.default_rng(seed + n)
    scn = Scene()
    prim = _quad(scn, -6.0, 6.0, -6.0, 6.0)
    E = np.zeros(3)
    reach = 1.0
    for i in range(n):
        a = _grid(min(0.9, (1.0 - 0.4 ** (1.0 / n)) * rng.uniform(0.7, 1.3)))
        e = (0.3 + 1.4 * (i + 0.5) / n) * np.array([1.0, 0.5, 0.8])
        scn.add_node(prim, _black(scn, a, e.astype(np.float32)), np.eye(4) + _tz(-0.1 * i))
        p = float(ah.p_closest(a))
        E += np.asarray(np.float32(e), np.float64) * p * reach
        reach *= 1.0 - p
    E += np.asarray(L, np.float64) * reach
    cam = Camera()
    cam.type = "orthographic"
    cam.eye, cam.center = np.array([0.0, 0.0, 4.0], np.float32), np.zeros(3, np.float32)
    cam.xmag = cam.ymag = 1.0
    cam.znear, cam.zfar = 0.1, 10.0
    scn.camera = cam
    return scn, E


def shadow_veils(n, seed=31):
    """synth_furnace_polyhedron (Lambert 0.8) lit by one directional light, environment intensity 0, and n black BLEND layers
    across the light's direction between the body and the light, outside the camera's view.  Every other layer is single-sided
    and faces away from the body (shadow rays do not cull).  Returns (scene, face normals, estcases case, factor): a face's
    expectation is the light-only one times factor = prod_i (1 - p_i), p on the shadow grid."""
    import estcases
    rng = np.random.default_rng(seed + n)
    case = dict(mat=estcases.LAMBERT(0.8), env="furnace", intensity=0.0, lights="shadow_veils")
    scn, normals = synth.synth_furnace_polyhedron([case["mat"]])
    scn.lights = [synth._light("directional", direction=SHADOW_LIGHT_DIR, color=(1.0, 0.95, 0.9), intensity=1.5)]
    to_light = -np.asarray(SHADOW_LIGHT_DIR, np.float64) / np.linalg.norm(SHADOW_LIGHT_DIR)
    e1 = np.cross(to_light, [0.0, 1.0, 0.0])
    e1 /= np.linalg.norm(e1)
    e2 = np.cross(to_light, e1)                       # e1 x e2 = to_light: the front face looks away from the body
    factor = 1.0
    for i in range(n):
        a = 0.0 if (i == 2 and n >= 5) else _grid(min(0.9, (1.0 - 0.75 ** (1.0 / n)) * rng.uniform(0.7, 1.3)))
        c = (5.0 + 0.1 * i) * to_light
        pos = [c - 1.5 * e1 - 1.5 * e2, c + 1.5 * e1 - 1.5 * e2, c + 1.5 * e1 + 1.5 * e2, c - 1.5 * e1 + 1.5 * e2]
        prim = scn.add_primitive(pos, [[0, 1, 2], [0, 2, 3]], normals=[to_light] * 4)
        scn.add_node(prim, _black(scn, a, double_sided=i % 2 == 0))
        factor *= 1.0 - float(ah.p_shadow(a))
    return scn, normals, case, factor


def veils_off_view(scn, first_node):
    """how far the render nodes from `first_node` on stay from the orthographic camera's axis: the least over them of (the
    distance of a quad's centre from the axis - its centre-to-corner distance), in units of the view's half-diagonal"""
    cam = scn.camera
    v = np.asarray(cam.eye, np.float64) - np.asarray(cam.center, np.float64)
    v /= np.linalg.norm(v)
    d = []
    for rn in scn.render_nodes[first_node:]:
        p = scn.render_prims[rn["renderPrimID"]]["positions"].astype(np.float64)
        c = p.mean(0)
        d.append(np.linalg.norm(c - (c @ v) * v) - np.linalg.norm(p - c, axis=1).max())
    return min(d) / math.hypot(cam.xmag, cam.ymag)
