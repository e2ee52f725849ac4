"""Scenes and rays for the tree-walk precision tests (tests/test_walk_precision.py on the host, tests/test_gpu_walk_precision.py on
the device), and the float64 classification of every (ray, triangle) pair they are held to.

The walks must return exactly what a brute force with the kernel's triangle test returns.  Where that is hard is a node far from
the ray origin relative to its own size: the rounding of the slab distances and of the triangle test grows with the distance, while
a node's quantum does not.  So the families put small triangles far from the origins (soups from 1e-3 to 1e4 units, offsets to 1e5,
triangles 1e-5 of the scene), flat nodes (coplanar tiles), boxes spanned by slivers, and coincident triangles; the rays hit interior,
edge and vertex points from 1 to 3e5 node sizes away, along the axes with +0 and -0 components, with components below the 1e-20
clamp of the walk, from origins on a triangle with tmin > 0, and as shadow segments that end at their hit and its fp32 neighbours.

Everything is generated from fixed seeds; triangles are stored as the flatten stores them (v0, fp32 v1 - v0, fp32 v2 - v0)."""
import numpy as np

F32 = np.float32
EPS = 2.0 ** -24  # unit roundoff of fp32
ETA = 2.0 ** -149  # absolute error bound of an fp32 rounding into the subnormal range


def _soup(rng, n, tri, scale=1.0, offset=0.0):
    c = (rng.random((n, 1, 3)) - 0.5) * 2
    return ((c + (rng.random((n, 3, 3)) - 0.5) * tri) * scale + offset).astype(F32)


def _layers():
    """Floor tiles: 12 coplanar layers of 16 x 16 axis-aligned quads (zero-thickness nodes), alternately z-up and y-up."""
    g = np.linspace(-1, 1, 17)
    out = []
    for k, h in enumerate(np.linspace(-0.9, 0.9, 12)):
        x0, y0 = np.meshgrid(g[:-1], g[:-1], indexing="ij")
        x0, y0 = x0.ravel(), y0.ravel()
        s = g[1] - g[0]
        p = np.stack([np.stack([x0, y0], 1), np.stack([x0 + s, y0], 1), np.stack([x0 + s, y0 + s], 1), np.stack([x0, y0 + s], 1)], 1)
        q = np.concatenate([p, np.full(p.shape[:2] + (1,), h)], 2)
        if k % 2:
            q = q[..., [0, 2, 1]]
        out += [q[:, [0, 1, 2]], q[:, [0, 2, 3]]]
    return np.concatenate(out).astype(F32)


def _slivers(rng, n=1500):
    """Long slivers spanning the scene (length ~2, width 1e-3 .. 1e-5) among a soup of ordinary triangles."""
    a = (rng.random((n, 3)) - 0.5) * 2
    b = -a + (rng.random((n, 3)) - 0.5) * 0.2
    w = (rng.normal(size=(n, 3))) * 10.0 ** rng.uniform(-5, -3, (n, 1))
    sl = np.stack([a, b, a + 0.5 * (b - a) + w], 1)
    return np.concatenate([sl, _soup(rng, 2500, 0.3)]).astype(F32)


def _duplicates(rng):
    """A soup in which 400 triangles appear three times at the same place (ties in t broken by id)."""
    t = _soup(rng, 3200, 0.3)
    return np.concatenate([t, t[:400], t[:400]]).astype(F32)


# name -> (triangles, size of one triangle, i.e. of a leaf node)
def _families():
    fam = {}
    for seed, (name, tri, scale, off) in enumerate((("soup_1e-3", 0.3, 1e-3, 0.0), ("soup_1", 0.3, 1.0, 0.0), ("soup_1e4", 0.3, 1e4, 0.0),
                                                    ("soup_1e4_at_1e5", 0.3, 1e4, 1e5), ("soup_1_at_1e5", 0.3, 1.0, 1e5),
                                                    ("tiny_1e-5", 2e-5, 1.0, 0.0))):
        fam[name] = (lambda seed=seed, tri=tri, scale=scale, off=off: _soup(np.random.default_rng(seed), 4000, tri, scale, off), tri * scale)
    fam["layers"] = (_layers, 0.125)
    fam["slivers"] = (lambda: _slivers(np.random.default_rng(11)), 0.3)
    fam["duplicates"] = (lambda: _duplicates(np.random.default_rng(13)), 0.3)
    return fam


FAMILIES = tuple(_families())


def records(v):
    """(n, 3, 3) fp32 vertices -> (n, 9) (v0, e1, e2) exactly as the flatten computes them (fp32 differences)"""
    v = np.asarray(v, F32)
    return np.concatenate([v[:, 0], v[:, 1] - v[:, 0], v[:, 2] - v[:, 0]], 1)


def _unit(d):
    return d / np.linalg.norm(d, axis=1, keepdims=True)


def _aim_points(rng, v, n):
    """n points on random triangles: a third interior, a third on an edge (one barycentric exactly 0), a third on a vertex"""
    k = rng.integers(0, len(v), n)
    b = rng.random((n, 3))
    kind = np.arange(n) % 3
    b[kind == 1, rng.integers(0, 3, n)[kind == 1]] = 0.0
    vert = np.eye(3)[rng.integers(0, 3, n)]
    b[kind == 2] = vert[kind == 2]
    b /= b.sum(1, keepdims=True)
    return k, np.einsum("nk,nkd->nd", b, v[k].astype(np.float64))


def rays(v, leaf, n=3000, seed=5):
    """(n, 8) fp32 rays (o, tmin, d, tmax) at the triangles v, whose leaves are about `leaf` wide: nine groups (module docstring)"""
    rng = np.random.default_rng(seed)
    R = np.zeros((n, 8), F32)
    R[:, 7] = 1e30
    g = np.arange(n) % 9
    _, p = _aim_points(rng, v, n)
    # distance to the origin: 1 .. 3e5 leaf sizes (bounded so the origin stays within fp32 reach of the scene)
    dist = leaf * 10.0 ** rng.uniform(0, 5.5, n)
    d = _unit(rng.normal(size=(n, 3)))
    # groups 0-2: aimed at interior / edge / vertex points (the aim points cycle through the three kinds)
    # group 3: axis-parallel, the other components +0 or -0
    ax = rng.integers(0, 3, n)
    sgn = rng.choice([-1.0, 1.0], n)
    zero = np.where(rng.random((n, 3)) < 0.5, -0.0, 0.0)
    axd = zero.copy()
    axd[np.arange(n), ax] = sgn
    # group 4: components below the walk's 1e-20 clamp (and subnormal ones)
    tiny = axd.copy()
    tiny[axd == 0] = rng.choice([1e-21, -1e-25, 1e-38, -1e-44, 0.0, -0.0], (axd == 0).sum())
    d = np.where((g == 3)[:, None], axd, d)
    d = np.where((g == 4)[:, None], tiny, d)
    o = p - d * dist[:, None]
    R[:, 0:3] = o
    R[:, 4:7] = d
    # groups 5-6: origins on a triangle (the aim point itself), random direction, tmin > 0
    on = (g == 5) | (g == 6)
    R[on, 0:3] = p[on]
    R[on, 4:7] = _unit(rng.normal(size=(on.sum(), 3)))
    R[on, 3] = (leaf * 10.0 ** rng.uniform(-4, -1, on.sum())).astype(F32)
    # groups 7-8: shadow segments ending at the aim point's t and its fp32 neighbours (the kernel's t is within a few ulp of it)
    seg = (g == 7) | (g == 8)
    t64 = np.einsum("nd,nd->n", p - R[:, 0:3].astype(np.float64), R[:, 4:7].astype(np.float64)) / np.einsum("nd,nd->n", R[:, 4:7], R[:, 4:7])
    t32 = t64[seg].astype(F32)
    steps = rng.integers(-2, 3, seg.sum())
    tm = t32.copy()
    for s in range(2):
        up, dn = steps > s, steps < -s
        tm[up] = np.nextafter(tm[up], F32(np.inf))
        tm[dn] = np.nextafter(tm[dn], F32(0))
    R[seg, 7] = tm
    return R


def case(name):
    """(fp32 vertices (n, 3, 3), rays (m, 8)) of one family"""
    build, leaf = _families()[name]
    v = build()
    return v, rays(v, leaf)


def dump(path, v, R):
    """the host checkers' input file: counts, (v0, e1, e2) per triangle, 8 floats per ray"""
    tr = records(v)
    with open(path, "wb") as f:
        f.write(np.array([len(tr), len(R)], np.uint32).tobytes())
        f.write(np.ascontiguousarray(tr, F32).tobytes())
        f.write(np.ascontiguousarray(R, F32).tobytes())


def read_hits(path):
    """brute-force hits written by host_traverse_check: int (ray, gid) and float (t, u, v, det) columns"""
    a = np.fromfile(path, np.float32).reshape(-1, 6)
    return a[:, :2].view(np.uint32).astype(np.int64), a[:, 2:]


def _gamma(k):
    return k * EPS / (1 - k * EPS)


def classify(rec, R, chunk=50):
    """Float64 classification of every (ray, triangle) pair against the kernel's fp32 triangle test (Moeller-Trumbore as
    traverse.cuh's fma chain).  The triangle is the stored one (v0, v0 + e1, v0 + e2) and the ray the fp32 ray, both widened
    to float64, so the exact quantities are det = e1.(d x e2), nu = tvec.(d x e2), nv = d.(tvec x e1), nt = e2.(tvec x e1)
    with tvec = o - v0.  The fp32 chain's error bound, from the a-priori bounds of its operations (Higham ch. 3, g_k = k e / (1 - k e)):
      tvec: one rounding; pvec = crossFma(d, e2): two; det: pvec's two and three more -> |det^ - det| <= g5 sum|e1| (|d||e2| + |d||e2|)
      nu, nv, nt: tvec's one, the cross product's two, the dot's three -> g6 times the same sums of absolute products
      u = nu^ * fl(1 / det^): two more relative roundings, and the quotient's sensitivity (|nu| Ed + Enu) / (|det| - Ed)
      u + v: one more rounding.
    Directions with subnormal components make products underflow: every sum above also gets 8 ETA times (1 + its operands' norm).
    A pair is a certain hit when every inequality of the test (det != 0, 0 <= u <= 1, v >= 0, u + v <= 1, tmin < t < tmax) holds
    with more than its bound to spare, a certain miss when one fails by more than its bound, otherwise borderline.
    A pair whose segment passes far from the triangle's box (_far) is a certain miss whatever its det.
    Returns the (ray, triangle) index pairs of the certain hits and of the borderline pairs, and the number of pairs; every other
    pair is a certain miss."""
    rec = np.asarray(rec, np.float64)
    v0, e1, e2 = rec[:, 0:3], rec[:, 3:6], rec[:, 6:9]
    hits, border = [], []
    for r0 in range(0, len(R), chunk):
        Rc = np.asarray(R[r0:r0 + chunk], np.float64)
        o, d = Rc[:, None, 0:3], Rc[:, None, 4:7]
        tmin, tmax = Rc[:, None, 3], Rc[:, None, 7]
        tv = o - v0[None]
        atv = np.abs(tv)

        def cross(a, b):
            return np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                             a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], -1)

        def across(a, b):
            return np.stack([a[..., 1] * b[..., 2] + a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] + a[..., 0] * b[..., 2],
                             a[..., 0] * b[..., 1] + a[..., 1] * b[..., 0]], -1)

        E1, E2 = np.broadcast_to(e1[None], tv.shape), np.broadcast_to(e2[None], tv.shape)
        D = np.broadcast_to(d, tv.shape)
        pv, apv = cross(D, E2), across(np.abs(D), np.abs(E2))
        qv, aqv = cross(tv, E1), across(atv, np.abs(E1))
        under = lambda a: 8 * ETA * (1 + np.abs(a).sum(-1))  # noqa: E731
        det, Ed = (E1 * pv).sum(-1), _gamma(5) * (np.abs(E1) * apv).sum(-1) + under(E1)
        nu, Enu = (tv * pv).sum(-1), _gamma(6) * (atv * apv).sum(-1) + under(tv)
        nv, Env = (D * qv).sum(-1), _gamma(6) * (np.abs(D) * aqv).sum(-1) + under(D)
        nt, Ent = (E2 * qv).sum(-1), _gamma(6) * (np.abs(E2) * aqv).sum(-1) + under(E2)
        sure = np.abs(det) > Ed
        with np.errstate(divide="ignore", invalid="ignore"):
            den = np.where(sure, np.abs(det) - Ed, 1.0)
            u, v, t = nu / det, nv / det, nt / det
            Eu = (np.abs(nu) / np.abs(det) * Ed + Enu) / den * (1 + _gamma(2)) + _gamma(2) * np.abs(u)
            Ev = (np.abs(nv) / np.abs(det) * Ed + Env) / den * (1 + _gamma(2)) + _gamma(2) * np.abs(v)
            Et = (np.abs(nt) / np.abs(det) * Ed + Ent) / den * (1 + _gamma(2)) + _gamma(2) * np.abs(t)
            Euv = (Eu + Ev) * (1 + EPS) + EPS * (np.abs(u) + np.abs(v))
            hit = sure & (u > Eu) & (u < 1 - Eu) & (v > Ev) & (u + v < 1 - Euv) & (t > tmin + Et) & (t < tmax - Et)
            miss = (det == 0) | (sure & ((u < -Eu) | (u > 1 + Eu) | (v < -Ev) | (u + v > 1 + Euv) | (t < tmin - Et) | (t > tmax + Et)))
        miss |= _far(Rc, rec)  # parallel or uncertain det: the pair is still a certain miss if the segment passes far from the box
        rr, tt = np.nonzero(hit)
        hits.append(np.stack([rr + r0, tt], 1))
        rr, tt = np.nonzero(~hit & ~miss)
        border.append(np.stack([rr + r0, tt], 1))
    return np.concatenate(hits), np.concatenate(border), len(R) * len(rec)


def _far(Rc, rec):
    """pairs whose ray segment misses the triangle's box by more than 1e-3 of the box's distance from the origin: the fp32
    triangle test errs by a few 1e-7 of that distance, and an exactly coplanar ray gets det = 0 (held by the tests)"""
    v0, e1, e2 = rec[:, 0:3], rec[:, 3:6], rec[:, 6:9]
    lo = np.minimum(v0, np.minimum(v0 + e1, v0 + e2))
    hi = np.maximum(v0, np.maximum(v0 + e1, v0 + e2))
    o, d = Rc[:, None, 0:3], Rc[:, None, 4:7]
    reach = np.abs(0.5 * (lo + hi)[None] - o).sum(-1) + (hi - lo).sum(-1)[None]
    pad = 1e-3 * reach
    with np.errstate(divide="ignore", invalid="ignore"):
        inv = 1.0 / d
        a = (lo[None] - pad[..., None] - o) * inv
        b = (hi[None] + pad[..., None] - o) * inv
        # a zero component gives +-inf inside the slab and nan on its face: fmin / fmax semantics drop the nan
        tn = np.fmax.reduce(np.fmin(a, b), -1)
        tf = np.fmin.reduce(np.fmax(a, b), -1)
    tn = np.maximum(tn, Rc[:, None, 3] * (1 - 1e-3))
    tf = np.minimum(tf, Rc[:, None, 7] * (1 + 1e-3))
    return tn > tf
