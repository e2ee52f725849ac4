"""Seeded procedural stand-ins for the BASELINE scenes that are not in the container.

The Khronos sample assets BASELINE.json names (Sponza, DamagedHelmet, DragonDispersion) are not
available offline (SURVEY.md §8d).  `synth_sponza` is the stand-in the survey specifies: a seeded
atrium of 262 144 instanced triangles, 25 materials, value-noise baseColor(sRGB) / metallic-roughness /
normal textures and ~10 % alpha-MASK foliage quads.  `synth_glass` is the transmission/volume case.
Everything is deterministic in `seed` so the oracle, the CUDA path and the bench see identical bytes.
"""
import math

import numpy as np

from .scene import Camera, Scene


# ------------------------------------------------------------------------------------------------
# mesh helpers
# ------------------------------------------------------------------------------------------------
def param_surface(f, nu, nv, uv_scale=(1.0, 1.0)):
    """Tessellate p = f(u, v), u,v in [0,1], into nu x nv quads (2 triangles each, CCW seen from +normal =
    dP/du x dP/dv).  Returns positions, normals, uv, tangents(w=+1), indices."""
    u = np.linspace(0.0, 1.0, nu + 1)
    v = np.linspace(0.0, 1.0, nv + 1)
    U, V = np.meshgrid(u, v, indexing="xy")  # [nv+1, nu+1]
    P = f(U, V)
    e = 1e-4
    du = (f(np.clip(U + e, 0, 1), V) - f(np.clip(U - e, 0, 1), V))
    dv = (f(U, np.clip(V + e, 0, 1)) - f(U, np.clip(V - e, 0, 1)))
    n = np.cross(du, dv)
    n /= np.maximum(np.linalg.norm(n, axis=-1, keepdims=True), 1e-20)
    t = du / np.maximum(np.linalg.norm(du, axis=-1, keepdims=True), 1e-20)
    t = t - n * np.sum(n * t, -1, keepdims=True)
    t /= np.maximum(np.linalg.norm(t, axis=-1, keepdims=True), 1e-20)
    pos = P.reshape(-1, 3).astype(np.float32)
    nrm = n.reshape(-1, 3).astype(np.float32)
    uv = np.stack([U * uv_scale[0], V * uv_scale[1]], -1).reshape(-1, 2).astype(np.float32)
    tan = np.concatenate([t.reshape(-1, 3), np.ones((pos.shape[0], 1))], 1).astype(np.float32)
    i0 = (np.arange(nv)[:, None] * (nu + 1) + np.arange(nu)[None, :]).reshape(-1)
    i1, i2, i3 = i0 + 1, i0 + (nu + 1), i0 + (nu + 2)
    idx = np.stack([np.stack([i0, i1, i3], 1), np.stack([i0, i3, i2], 1)], 1).reshape(-1, 3).astype(np.uint32)
    return pos, nrm, uv, tan, idx


def _xyz(x, y, z):
    return np.stack([x, y, z], -1)


def value_noise(size, octaves, rng, channels=1):
    """Tileable multi-octave value noise in [0,1], shape [size,size,channels]
    (smoothstep-interpolated random lattices, evaluated as two small matmuls per octave)."""
    out = np.zeros((channels, size, size), np.float32)
    amp, tot = 1.0, 0.0
    for o in range(octaves):
        n = 4 << o
        if n > size:
            break
        g = rng.random((channels, n, n)).astype(np.float32)
        x = np.arange(size, dtype=np.float32) * (n / size)
        x0 = np.floor(x).astype(np.int64)
        fx = x - x0
        fx = fx * fx * (3 - 2 * fx)
        W = np.zeros((size, n), np.float32)
        W[np.arange(size), x0 % n] += 1 - fx
        W[np.arange(size), (x0 + 1) % n] += fx
        out += amp * np.matmul(np.matmul(W, g), W.T)
        tot += amp
        amp *= 0.5
    return np.ascontiguousarray(np.moveaxis(out / tot, 0, -1))


def _u8(a):
    return np.clip(np.round(a * 255.0), 0, 255).astype(np.uint8)


def make_texture_set(size, rng, tint):
    """(baseColor sRGB RGBA8, metallicRoughness RGBA8 [G=rough,B=metal], normal RGBA8)."""
    h = value_noise(size, 7, rng, 1)[..., 0]
    detail = value_noise(size, 7, rng, 3)
    base = np.clip(np.asarray(tint, np.float32)[None, None, :] * (0.86 + 0.28 * h[..., None]) * (0.93 + 0.14 * detail), 0, 1)
    base_rgba = np.concatenate([_u8(base), np.full((size, size, 1), 255, np.uint8)], -1)
    rough = np.clip(0.35 + 0.6 * value_noise(size, 6, rng, 1)[..., 0], 0, 1)
    metal = (value_noise(size, 4, rng, 1)[..., 0] > 0.62).astype(np.float32) * 0.9
    mr = np.stack([np.ones_like(rough), rough, metal, np.ones_like(rough)], -1)
    # normal map from the height field (central differences, tileable)
    s = 6.0
    dx = (np.roll(h, -1, 1) - np.roll(h, 1, 1)) * s
    dy = (np.roll(h, -1, 0) - np.roll(h, 1, 0)) * s
    n = np.stack([-dx, -dy, np.ones_like(h)], -1)
    n /= np.linalg.norm(n, axis=-1, keepdims=True)
    nm = np.concatenate([_u8(n * 0.5 + 0.5), np.full((size, size, 1), 255, np.uint8)], -1)
    return base_rgba, _u8(mr), nm


def make_leaf_texture(size, rng):
    """Foliage atlas: green sRGB colour, alpha = leaf-shaped mask (MASK mode, cutoff 0.5)."""
    y, x = np.mgrid[0:size, 0:size].astype(np.float32) / size
    cells = 4
    cx, cy = (x * cells) % 1.0 - 0.5, (y * cells) % 1.0 - 0.5
    leaf = ((cx / 0.28) ** 2 + (cy / 0.45) ** 2) < 1.0
    vein = np.abs(cx) < 0.015
    n = value_noise(size, 6, rng, 3)
    col = np.clip(np.array([0.10, 0.42, 0.08], np.float32) * (0.6 + 0.9 * n), 0, 1)
    col[vein & leaf] *= 0.6
    alpha = leaf.astype(np.float32)
    return np.concatenate([_u8(col), _u8(alpha)[..., None]], -1)


# ------------------------------------------------------------------------------------------------
# SynthSponza
# ------------------------------------------------------------------------------------------------
def synth_sponza(seed=1234, tex_size=2048, tri_budget=262144, detail=1.0):
    """Procedural atrium stand-in for Sponza. `detail` scales tessellation (tests use < 1);
    with detail=1 the instanced triangle count is exactly `tri_budget`."""
    rng = np.random.default_rng(seed)
    scn = Scene()

    def q(n):  # tessellation scaled by detail, at least 2
        return max(2, int(round(n * math.sqrt(detail))))

    # ---- textures + 25 materials ----
    # sRGB tints; with the noise modulation the mean LINEAR albedo is ~0.5 (lit stone / fabric, like Sponza's textures),
    # so paths survive Russian roulette well past depth 3 and the depth-12 budget is actually exercised
    tints = [(0.88, 0.83, 0.74), (0.78, 0.71, 0.63), (0.72, 0.42, 0.32), (0.42, 0.52, 0.72), (0.90, 0.87, 0.83), (0.66, 0.66, 0.68)]
    tex_sets = []
    for t in tints:
        b, mr, nm = make_texture_set(tex_size, rng, t)
        tex_sets.append((scn.add_texture(b, srgb=True), scn.add_texture(mr), scn.add_texture(nm)))
    leaf_tex = scn.add_texture(make_leaf_texture(tex_size, rng), srgb=True)

    mats = []
    for m in range(24):
        ts = tex_sets[m % len(tex_sets)]
        uvs = 1.0 + (m % 3)
        xf = (uvs, 0, 0, uvs, 0.13 * m, 0.07 * m)
        kw = dict(
            pbrBaseColorFactor=[0.85 + 0.15 * rng.random(), 0.85 + 0.15 * rng.random(), 0.85 + 0.15 * rng.random(), 1.0],
            pbrRoughnessFactor=0.5 + 0.5 * rng.random(), pbrMetallicFactor=1.0 if m % 5 == 0 else 0.3 * rng.random(),
            pbrBaseColorTexture=scn.add_texture_info(ts[0], 0, xf),
            pbrMetallicRoughnessTexture=scn.add_texture_info(ts[1], 0, xf),
            normalTexture=scn.add_texture_info(ts[2], 0, xf), normalTextureScale=0.6 + 0.4 * rng.random(),
            doubleSided=1 if m % 4 == 1 else 0)
        if m == 7:
            kw.update(clearcoatFactor=1.0, clearcoatRoughness=0.05)
        if m == 11:
            kw.update(emissiveFactor=[1.5, 1.2, 0.8])
        mats.append(scn.add_material(**kw))
    leaf_mat = scn.add_material(pbrBaseColorFactor=[1, 1, 1, 1], pbrRoughnessFactor=0.6, pbrMetallicFactor=0.0,
                                alphaMode=1, alphaCutoff=0.5, doubleSided=1,
                                pbrBaseColorTexture=scn.add_texture_info(leaf_tex, 0))

    LX, LZ, H = 15.0, 6.0, 12.0

    def add(pos, nrm, uv, tan, idx, mat, matrix=None):
        p = scn.add_primitive(pos, idx, normals=nrm, uv0=uv, tangents=tan)
        scn.add_node(p, mat, matrix)
        return p

    def T(x, y, z, s=1.0, ry=0.0):
        c, sn = math.cos(ry), math.sin(ry)
        return np.array([[c * s, 0, sn * s, x], [0, s, 0, y], [-sn * s, 0, c * s, z], [0, 0, 0, 1]], np.float64)

    # floor (slightly bumpy), normal up
    def floor_f(u, v):
        x, z = (u * 2 - 1) * LX, (1 - v * 2) * LZ
        return _xyz(x, 0.03 * np.sin(x * 3.0) * np.sin(z * 2.5), z)
    add(*param_surface(floor_f, q(128), q(64), (10, 4)), mats[0])

    # long walls (z = -LZ facing +z, z = +LZ facing -z), short walls
    def wall_zm(u, v):
        return _xyz((u * 2 - 1) * LX, v * H, np.full_like(u, -LZ) + 0.05 * np.sin(u * 40) * np.sin(v * 25))
    def wall_zp(u, v):
        return _xyz((1 - u * 2) * LX, v * H, np.full_like(u, LZ) - 0.05 * np.sin(u * 40) * np.sin(v * 25))
    def wall_xm(u, v):
        return _xyz(np.full_like(u, -LX), v * H, (1 - u * 2) * LZ)
    def wall_xp(u, v):
        return _xyz(np.full_like(u, LX), v * H, (u * 2 - 1) * LZ)
    add(*param_surface(wall_zm, q(64), q(32), (8, 3)), mats[1])
    add(*param_surface(wall_zp, q(64), q(32), (8, 3)), mats[2])
    add(*param_surface(wall_xm, q(32), q(32), (3, 3)), mats[3])
    add(*param_surface(wall_xp, q(32), q(32), (3, 3)), mats[4])

    # ceiling ring with an open slot (so the environment lights the atrium), normal down
    def ceil_a(u, v):
        return _xyz((u * 2 - 1) * LX, np.full_like(u, H), -LZ + v * (LZ * 0.55))
    def ceil_b(u, v):
        return _xyz((1 - u * 2) * LX, np.full_like(u, H), LZ - v * (LZ * 0.55))
    add(*param_surface(ceil_a, q(64), q(16), (8, 1)), mats[5])
    add(*param_surface(ceil_b, q(64), q(16), (8, 1)), mats[6])

    # columns: one primitive, 48 instances (two rows, two storeys)
    def column_f(u, v):
        r = 0.35 * (1.0 + 0.12 * np.cos(u * 2 * math.pi * 12) * (v > 0.08) * (v < 0.92)) * (1.0 + 0.5 * (np.abs(v - 0.5) > 0.46))
        a = u * 2 * math.pi
        return _xyz(r * np.cos(a), v * 4.5, -r * np.sin(a))
    cp = scn.add_primitive(*[x for x in _split(param_surface(column_f, q(32), q(16), (2, 4)))])
    k = 0
    for storey in range(2):
        for row in (-1, 1):
            for c in range(12):
                x = -LX + 1.8 + c * (2 * LX - 3.6) / 11
                scn.add_node(cp, mats[8 + (k % 4)], T(x, storey * 5.2, row * (LZ - 1.6), 1.0, 0.37 * k))
                k += 1

    # gallery slabs (upper floor) along both long sides
    def slab(zc):
        def f(u, v):
            return _xyz((u * 2 - 1) * LX, np.full_like(u, 4.9) + 0.02 * np.sin(u * 60), zc + (0.5 - v) * 2.6)
        return f
    add(*param_surface(slab(-(LZ - 1.3)), q(64), q(8), (8, 1)), mats[12])
    add(*param_surface(slab(LZ - 1.3), q(64), q(8), (8, 1)), mats[13])

    # curtains: displaced cloth panels hanging in the arcades
    def curtain(phase):
        def f(u, v):
            return _xyz((u - 0.5) * 2.2, 4.6 - v * 3.6, 0.18 * np.sin(u * 2 * math.pi * 3 + phase) * (0.3 + v))
        return f
    for c in range(8):
        pos, nrm, uv, tan, idx = param_surface(curtain(1.7 * c), q(64), q(64), (2, 3))
        p = scn.add_primitive(pos, idx, normals=nrm, uv0=uv, tangents=tan)
        side = -1 if c % 2 == 0 else 1
        scn.add_node(p, mats[14 + (c % 4)], T(-LX + 4.0 + (c // 2) * 7.3, 0.0, side * (LZ - 1.65), 1.0, 0.0 if side > 0 else math.pi))

    # vases / spheres: one primitive, 16 instances
    def vase_f(u, v):
        th = v * math.pi
        r = 0.55 * np.sin(th) * (1.0 + 0.25 * np.sin(v * 9.0)) + 0.02
        a = u * 2 * math.pi
        return _xyz(r * np.cos(a), 0.9 - 0.9 * np.cos(th), -r * np.sin(a))
    vp = scn.add_primitive(*[x for x in _split(param_surface(vase_f, q(64), q(32), (3, 2)))])
    for c in range(16):
        x = -LX + 2.5 + (c % 8) * (2 * LX - 5.0) / 7
        z = -1.8 if c < 8 else 1.8
        scn.add_node(vp, mats[18 + (c % 6)], T(x, 0.0, z, 0.8 + 0.4 * rng.random(), rng.random() * 6.28))

    # filler rubble strip down the middle: sized so the total hits the budget exactly (detail == 1)
    def tri_total():
        return scn.num_triangles()
    foliage_quads = int(round(tri_budget * 0.10 / 2 * detail))
    remaining = int(tri_budget * detail) - tri_total() - foliage_quads * 2
    if remaining >= 8:
        nv_ = 8
        nu_ = max(1, remaining // (2 * nv_))
        def rubble(u, v):
            x, z = (u * 2 - 1) * (LX - 2), (v - 0.5) * 1.6
            return _xyz(x, 0.05 + 0.12 * np.abs(np.sin(x * 5.0) * np.cos(z * 7.0)), -z)
        add(*param_surface(rubble, nu_, nv_, (12, 1)), mats[7])
        left = int(tri_budget * detail) - tri_total() - foliage_quads * 2
        foliage_quads += max(0, left) // 2

    # foliage: alpha-masked double-sided quads in clumps around the vases (MASK, ~10 % of triangles)
    per_prim = 1024
    done = 0
    while done < foliage_quads:
        nq = min(per_prim, foliage_quads - done)
        vi = rng.integers(0, 16, nq)
        vx = -LX + 2.5 + (vi % 8) * (2 * LX - 5.0) / 7
        vz = np.where(vi < 8, -1.8, 1.8)
        c = np.stack([vx, np.full(nq, 2.1), vz], 1) + rng.normal(size=(nq, 3)) * np.array([0.55, 0.45, 0.55])
        ax = rng.normal(size=(nq, 3))
        ax /= np.linalg.norm(ax, axis=1, keepdims=True)
        bx = np.cross(ax, rng.normal(size=(nq, 3)))
        bx /= np.linalg.norm(bx, axis=1, keepdims=True)
        sz = 0.10 + 0.12 * rng.random((nq, 1))
        corners = np.stack([c - ax * sz - bx * sz, c + ax * sz - bx * sz, c + ax * sz + bx * sz, c - ax * sz + bx * sz], 1)
        nrm = np.repeat(np.cross(ax, bx)[:, None, :], 4, 1)
        cell = rng.integers(0, 4, (nq, 2)).astype(np.float32) * 0.25
        uv = np.stack([cell, cell + [0.25, 0], cell + [0.25, 0.25], cell + [0, 0.25]], 1)
        base = (np.arange(nq) * 4)[:, None]
        idx = np.concatenate([base + [0, 1, 2], base + [0, 2, 3]], 1).reshape(-1, 3)
        p = scn.add_primitive(corners.reshape(-1, 3), idx, normals=nrm.reshape(-1, 3), uv0=uv.reshape(-1, 2))
        scn.add_node(p, leaf_mat)
        done += nq

    cam = Camera()
    cam.eye = np.array([-LX + 1.5, 2.2, 0.4], np.float32)
    cam.center = np.array([LX - 2.0, 4.0, -0.3], np.float32)
    cam.up = np.array([0, 1, 0], np.float32)
    cam.yfov = math.radians(60.0)
    cam.znear, cam.zfar = 0.05, 200.0
    scn.camera = cam
    return scn


def _split(t):
    pos, nrm, uv, tan, idx = t
    return [pos, idx, nrm, uv, None, tan, None]


# ------------------------------------------------------------------------------------------------
# SynthGlass: transmission + volume stand-in for DragonDispersion
# ------------------------------------------------------------------------------------------------
def synth_glass(seed=1234, n=96, scatter=False, dispersion=0.0):
    rng = np.random.default_rng(seed)
    scn = Scene()
    k = rng.random(6) * 6.28

    def blob(u, v):
        th, a = v * math.pi, u * 2 * math.pi
        r = 1.0 + 0.12 * np.sin(3 * a + k[0]) * np.sin(4 * th + k[1]) + 0.06 * np.sin(7 * a + k[2]) * np.sin(5 * th + k[3])
        return _xyz(r * np.sin(th) * np.cos(a), 1.15 - r * np.cos(th), -r * np.sin(th) * np.sin(a))
    pos, nrm, uv, tan, idx = param_surface(blob, n, n // 2, (1, 1))
    glass = scn.add_material(pbrBaseColorFactor=[1, 1, 1, 1], pbrRoughnessFactor=0.05, pbrMetallicFactor=0.0,
                             transmissionFactor=1.0, thicknessFactor=1.0, attenuationDistance=0.5,
                             attenuationColor=[0.85, 0.35, 0.25], ior=1.5,
                             multiscatterColorFactor=[0.6, 0.6, 0.6] if scatter else [0, 0, 0], scatterAnisotropy=0.3, dispersion=dispersion)
    scn.add_node(scn.add_primitive(pos, idx, normals=nrm, uv0=uv, tangents=tan), glass)

    def ground(u, v):
        return _xyz((u * 2 - 1) * 6, np.zeros_like(u), (1 - v * 2) * 6)
    gp, gn, guv, gt, gi = param_surface(ground, 8, 8, (4, 4))
    gm = scn.add_material(pbrBaseColorFactor=[0.6, 0.6, 0.6, 1], pbrRoughnessFactor=0.7, pbrMetallicFactor=0.0)
    scn.add_node(scn.add_primitive(gp, gi, normals=gn, uv0=guv, tangents=gt), gm)
    cam = Camera()
    cam.eye = np.array([0.0, 1.8, 4.2], np.float32)
    cam.center = np.array([0.0, 1.0, 0.0], np.float32)
    cam.yfov = math.radians(45.0)
    cam.znear, cam.zfar = 0.05, 100.0
    scn.camera = cam
    return scn


def synth_layers(seed=1234, layers=14, tex_size=64, blend=False, tinted=False):
    """`layers` parallel quads in front of a floor: MASK (or BLEND) noise alpha, optionally a stack of thin tinted
    glass sheets.  Every camera / shadow ray meets more non-opaque candidates than one any-hit walk collects, so
    the continuation rounds and the final in-kernel fallback of the any-hit kernels all run."""
    rng = np.random.default_rng(seed)
    scn = Scene()
    a = value_noise(tex_size, 4, rng, 1)[..., 0]
    rgba = np.concatenate([_u8(np.stack([0.3 + 0.6 * a, 0.8 - 0.5 * a, 0.4 + 0.2 * a], -1)), _u8(np.clip(a * 1.6 - 0.25, 0, 1))[..., None]], -1)
    tex = scn.add_texture(rgba, srgb=True)
    if tinted:
        mat = scn.add_material(pbrBaseColorFactor=[0.9, 0.95, 0.8, 1], pbrRoughnessFactor=0.1, pbrMetallicFactor=0.0, transmissionFactor=0.9,
                               thicknessFactor=0.0, ior=1.2, doubleSided=1)
    else:
        mat = scn.add_material(pbrBaseColorFactor=[1, 1, 1, 1], pbrRoughnessFactor=0.8, pbrMetallicFactor=0.0, alphaMode=2 if blend else 1,
                               alphaCutoff=0.5, doubleSided=1, pbrBaseColorTexture=scn.add_texture_info(tex, 0))
    for l in range(layers):
        z = -0.15 * l

        def quad(u, v, z=z, l=l):
            return _xyz((u * 2 - 1) * 1.5 + 0.03 * l, 0.1 + v * 2.0, np.full_like(u, z))
        pos, nrm, uv, tan, idx = param_surface(quad, 3, 3, (1.0 + 0.37 * l, 1.0 + 0.21 * l))
        scn.add_node(scn.add_primitive(pos, idx, normals=nrm, uv0=uv, tangents=tan), mat)

    def ground(u, v):
        return _xyz((u * 2 - 1) * 5, np.zeros_like(u), (1 - v * 2) * 5)
    gp, gn, guv, gt, gi = param_surface(ground, 4, 4, (2, 2))
    gm = scn.add_material(pbrBaseColorFactor=[0.7, 0.7, 0.7, 1], pbrRoughnessFactor=0.9, pbrMetallicFactor=0.0)
    scn.add_node(scn.add_primitive(gp, gi, normals=gn, uv0=guv, tangents=gt), gm)
    cam = Camera()
    cam.eye = np.array([0.4, 1.3, 3.0], np.float32)
    cam.center = np.array([0.0, 1.0, -1.0], np.float32)
    cam.yfov = math.radians(50.0)
    cam.znear, cam.zfar = 0.05, 100.0
    scn.camera = cam
    return scn


def sampler_layers(seed=1234):
    """synth_layers with a texture and sampler of its own on each of 14 stacked alpha layers: non-power-of-two, N x 1 and
    1 x N images, CLAMP_TO_EDGE and MIRRORED_REPEAT (mixed per axis), NEAREST and LINEAR magnification, uv ranges far
    outside [0, 1], one layer on TEXCOORD_1, one KHR_materials_pbrSpecularGlossiness layer (diffuse-texture alpha), one with
    vertex-colour alpha and one BLEND layer.  Rays meet more candidates than one any-hit walk collects, so both the
    pre-gathered alpha records and the generic in-kernel alpha test run on every sampler state."""
    rng = np.random.default_rng(seed)
    scn = Scene()
    R, C, M = 10497, 33071, 33648
    # (w, h, wrapS, wrapT, magFilter, uv scale, uv offset, variant)
    layers = [(37, 23, R, R, 9729, (3.7, 2.1), (0.2, -0.4), None), (5, 3, C, M, 9728, (2.5, 3.5), (-0.7, -1.2), None),
              (64, 1, M, C, 9729, (3.0, 2.0), (-1.0, -0.5), None), (23, 37, M, M, 9728, (16.0, 12.0), (-7.0, -5.0), None),
              (16, 16, C, C, 9729, (5.0, 5.0), (-2.0, -2.0), None), (9, 17, R, M, 9728, (1.0, 1.0), (0.0, 0.0), "uv1"),
              (7, 7, C, R, 9729, (2.2, 1.7), (-0.6, 0.3), "specgloss"), (33, 5, R, C, 9728, (1.3, 2.4), (0.1, -0.7), "color"),
              (37, 23, M, R, 9729, (2.9, 1.9), (-1.1, 0.4), "blend"), (1, 7, R, M, 9729, (1.0, 3.3), (0.0, -1.4), None),
              (128, 64, R, R, 9729, (1.5, 1.5), (0.0, 0.0), None), (3, 5, M, M, 9728, (40.0, 40.0), (-13.0, -17.0), None),
              (6, 6, C, C, 9729, (3.0, 3.0), (-1.0, -1.0), None), (11, 2, M, M, 9728, (6.0, 4.0), (-2.5, -1.5), None)]
    for l, (w, h, ws, wt, mag, sc, off, variant) in enumerate(layers):
        rgba = rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
        tex = scn.add_texture(rgba, srgb=True, wrapS=ws, wrapT=wt, magFilter=mag, minFilter=9987 if mag == 9729 else 9984)
        ti = scn.add_texture_info(tex, 1 if variant == "uv1" else 0)
        if variant == "specgloss":
            mat = scn.add_material(pbrModel=1, pbrDiffuseFactor=[0.8, 0.7, 0.6, 1], pbrSpecularFactor=[0.04, 0.04, 0.04], pbrGlossinessFactor=0.3,
                                   alphaMode=1, alphaCutoff=0.5, doubleSided=1, pbrDiffuseTexture=ti)
        else:
            mat = scn.add_material(pbrBaseColorFactor=[1, 1, 1, 1], pbrRoughnessFactor=0.8, pbrMetallicFactor=0.0, alphaMode=2 if variant == "blend" else 1,
                                   alphaCutoff=0.5 if variant != "color" else 0.3, doubleSided=1, pbrBaseColorTexture=ti)

        def quad(u, v, z=-0.15 * l, l=l):
            return _xyz((u * 2 - 1) * 1.5 + 0.03 * l, 0.1 + v * 2.0, np.full_like(u, z))
        pos, nrm, uv, tan, idx = param_surface(quad, 3, 3)
        uv = (uv * np.float32(sc) + np.float32(off)).astype(np.float32)
        uv1, col = None, None
        if variant == "uv1":
            uv1, uv = uv * np.float32(3.1) - np.float32(1.2), uv[:, ::-1].copy()
        if variant == "color":
            a = _u8(rng.random(len(pos))).astype(np.uint32)
            col = np.uint32(0x00FFFFFF) | (a << 24)
        scn.add_node(scn.add_primitive(pos, idx, normals=nrm, uv0=uv, uv1=uv1, tangents=tan, colors=col), mat)

    def ground(u, v):
        return _xyz((u * 2 - 1) * 5, np.zeros_like(u), (1 - v * 2) * 5)
    gp, gn, guv, gt, gi = param_surface(ground, 4, 4, (2, 2))
    gm = scn.add_material(pbrBaseColorFactor=[0.7, 0.7, 0.7, 1], pbrRoughnessFactor=0.9, pbrMetallicFactor=0.0)
    scn.add_node(scn.add_primitive(gp, gi, normals=gn, uv0=guv, tangents=gt), gm)
    cam = Camera()
    cam.eye = np.array([0.4, 1.3, 3.0], np.float32)
    cam.center = np.array([0.0, 1.0, -1.0], np.float32)
    cam.yfov = math.radians(50.0)
    cam.znear, cam.zfar = 0.05, 100.0
    scn.camera = cam
    return scn


def synth_helmet(seed=1234, tex_size=2048):
    """Stand-in for DamagedHelmet (BASELINE config 2; the Khronos asset is not available offline): ONE mesh of 46 080 triangles with
    ONE material that binds base colour (sRGB), metallic-roughness, normal and emissive textures of tex_size^2, floating in the
    environment (no floor), camera framing it like the sample viewer does."""
    rng = np.random.default_rng(seed)
    scn = Scene()
    k = rng.random(8) * 6.28

    def shell(u, v):
        th, a = v * math.pi, u * 2 * math.pi
        r = 1.0 + 0.10 * np.sin(4 * a + k[0]) * np.sin(3 * th + k[1]) + 0.05 * np.sin(9 * a + k[2]) * np.sin(7 * th + k[3]) + 0.02 * np.sin(23 * a + k[4]) * np.sin(19 * th + k[5])
        return _xyz(r * np.sin(th) * np.cos(a), -r * np.cos(th), -r * np.sin(th) * np.sin(a) * 1.15)
    pos, nrm, uv, tan, idx = param_surface(shell, 160, 144, (2, 1))
    assert len(idx) == 46080
    base, mr, nm = make_texture_set(tex_size, rng, (0.62, 0.58, 0.52))
    em = np.zeros((tex_size, tex_size, 4), np.uint8)
    glow = value_noise(tex_size, 5, rng, 1)[..., 0] > 0.72
    em[glow] = (40, 160, 255, 255)
    em[..., 3] = 255
    mat = scn.add_material(pbrBaseColorFactor=[1, 1, 1, 1], pbrRoughnessFactor=1.0, pbrMetallicFactor=1.0, emissiveFactor=[1.0, 1.0, 1.0],
                           pbrBaseColorTexture=scn.add_texture_info(scn.add_texture(base, srgb=True)),
                           pbrMetallicRoughnessTexture=scn.add_texture_info(scn.add_texture(mr)),
                           normalTexture=scn.add_texture_info(scn.add_texture(nm)),
                           emissiveTexture=scn.add_texture_info(scn.add_texture(em, srgb=True)))
    scn.add_node(scn.add_primitive(pos, idx, normals=nrm, uv0=uv, tangents=tan), mat)
    cam = Camera()
    cam.eye = np.array([0.0, 0.3, 3.4], np.float32)
    cam.center = np.array([0.0, 0.0, 0.0], np.float32)
    cam.yfov = math.radians(45.0)
    cam.znear, cam.zfar = 0.05, 100.0
    scn.camera = cam
    return scn


def _sphere(cx, cy, cz, r, n=24, uv_scale=(2, 1)):
    def f(u, v):
        th, a = v * math.pi, u * 2 * math.pi
        return _xyz(cx + r * np.sin(th) * np.cos(a), cy - r * np.cos(th), cz - r * np.sin(th) * np.sin(a))
    return param_surface(f, n, n // 2, uv_scale)


def _light(kind, position=(0, 0, 0), direction=(0, -1, 0), color=(1, 1, 1), intensity=1.0, radius=0.0, rng=0.0, inner=0.0, outer=math.pi / 4,
           angular_size=0.0):
    """GltfLight the way SceneVk::updateRenderLightsBuffer fills it (src/gltf_scene_vk.cpp:1354-1394): type 1 directional
    (angularSizeOrInvRange = angular size), 2 spot, 3 point (angularSizeOrInvRange = 1 / range)."""
    from . import abi
    L = abi.Light()
    d = np.asarray(direction, np.float64)
    d = d / np.linalg.norm(d)
    L.direction[:] = d.tolist()
    L.position[:] = list(position)
    L.color[:] = list(color)
    L.intensity = intensity
    L.radius = radius
    L.type = {"directional": 1, "spot": 2, "point": 3}[kind]
    L.innerAngle, L.outerAngle = inner, outer
    L.angularSizeOrInvRange = angular_size if kind == "directional" else (1.0 / rng if rng > 0 else 0.0)
    return L


def synth_lit(seed=1234, tex_size=64):
    """Punctual lights (KHR_lights_punctual as the reference uploads them): a point light with radius 0 and one with a radius
    (sphere light, sampled), a spot light with a range, a directional light with and one without angular size, over a textured
    floor with three spheres (dielectric, metal, clearcoat).  Exercises sampleLights' light branch, singleLightContribution,
    the light/environment technique MIS and shadow rays of finite length (FEAT_LIGHTS)."""
    rng = np.random.default_rng(seed)
    scn = Scene()
    base, mr, nm = make_texture_set(tex_size, rng, (0.75, 0.7, 0.6))
    tb, tm, tn = scn.add_texture(base, srgb=True), scn.add_texture(mr), scn.add_texture(nm)
    floor = scn.add_material(pbrBaseColorFactor=[1, 1, 1, 1], pbrRoughnessFactor=1.0, pbrMetallicFactor=0.2,
                             pbrBaseColorTexture=scn.add_texture_info(tb), pbrMetallicRoughnessTexture=scn.add_texture_info(tm),
                             normalTexture=scn.add_texture_info(tn))

    def ground(u, v):
        return _xyz((u * 2 - 1) * 5, np.zeros_like(u), (1 - v * 2) * 5)
    scn.add_node(scn.add_primitive(*_split(param_surface(ground, 6, 6, (3, 3)))), floor)
    mats = [scn.add_material(pbrBaseColorFactor=[0.8, 0.25, 0.2, 1], pbrRoughnessFactor=0.45, pbrMetallicFactor=0.0),
            scn.add_material(pbrBaseColorFactor=[0.95, 0.8, 0.4, 1], pbrRoughnessFactor=0.25, pbrMetallicFactor=1.0),
            scn.add_material(pbrBaseColorFactor=[0.1, 0.3, 0.7, 1], pbrRoughnessFactor=0.6, pbrMetallicFactor=0.0, clearcoatFactor=1.0, clearcoatRoughness=0.05)]
    for k, m in enumerate(mats):
        scn.add_node(scn.add_primitive(*_split(_sphere(-1.6 + 1.6 * k, 0.6, 0.2 * k, 0.6))), m)
    scn.lights = [
        _light("point", position=(-2.0, 2.2, 1.5), color=(1.0, 0.9, 0.8), intensity=18.0),
        _light("point", position=(1.5, 1.6, 1.8), color=(0.6, 0.8, 1.0), intensity=12.0, radius=0.25),
        _light("spot", position=(0.0, 3.5, 0.5), direction=(0.1, -1.0, -0.1), color=(1, 1, 1), intensity=40.0, rng=9.0, inner=0.25, outer=0.55),
        _light("directional", direction=(-0.4, -1.0, -0.3), color=(1.0, 0.95, 0.9), intensity=1.5, angular_size=0.06),
        _light("directional", direction=(0.6, -0.7, 0.2), color=(0.4, 0.5, 0.7), intensity=0.7),
    ]
    cam = Camera()
    cam.eye = np.array([0.3, 2.2, 5.0], np.float32)
    cam.center = np.array([0.0, 0.5, 0.0], np.float32)
    cam.yfov = math.radians(45.0)
    cam.znear, cam.zfar = 0.05, 100.0
    scn.camera = cam
    return scn


def synth_material_zoo(seed=1234, tex_size=64, samplers=False):
    """One sphere per KHR_materials_* extension, every extension WITH its textures (all 22 slots of GltfShadeMaterial that
    the path tracer reads are bound somewhere; gltf_material_eval.h.slang:168-457), plus KHR_texture_transform, TEXCOORD_1 and
    vertex colours: sheen, iridescence (+ thickness texture), anisotropy (+ direction texture), specular / specular colour,
    clearcoat (+ roughness + normal), transmission texture + thickness texture (volume), diffuse transmission (+ colour),
    pbrSpecularGlossiness, emissive texture, BLEND alpha.  Runs the FEAT_ALL shade variant.
    samplers=True: the shared base-colour texture is a non-power-of-two crop with CLAMP_TO_EDGE x MIRRORED_REPEAT under a
    rotated and scaled KHR_texture_transform, and the metallic-roughness texture is sampled NEAREST (mip mode included)."""
    rng = np.random.default_rng(seed)
    scn = Scene()

    def noise_rgba(srgb=False, lo=0.15, hi=1.0, alpha=None):
        n = value_noise(tex_size, 5, rng, 4)
        a = lo + (hi - lo) * n
        if alpha is not None:
            a[..., 3] = alpha
        return scn.add_texture(_u8(a), srgb=srgb)
    base, mr, nm = make_texture_set(tex_size, rng, (0.8, 0.8, 0.8))
    xf = (0.8, 0.3, -0.3, 0.8, 0.1, 0.2)  # KHR_texture_transform as the 2x3 matrix the loader would write
    if samplers:
        t_base = scn.add_texture(base[:tex_size * 3 // 5, :tex_size - 7], srgb=True, wrapS=33071, wrapT=33648)
        t_mr, t_nm = scn.add_texture(mr, magFilter=9728, minFilter=9986), scn.add_texture(nm)
        c, s_ = 2.5 * math.cos(0.5), 2.5 * math.sin(0.5)
        base_xf = (c, s_ * 0.6, -s_, c * 0.6, -0.7, 0.4)   # rotation, scale (2.5, 1.5), offset
    else:
        t_base, t_mr, t_nm = scn.add_texture(base, srgb=True), scn.add_texture(mr), scn.add_texture(nm)
        base_xf = None

    def ti(tex, texcoord=0, transform=False):
        if tex == t_base and base_xf is not None:
            return scn.add_texture_info(tex, texcoord, base_xf)
        return scn.add_texture_info(tex, texcoord, xf if transform else (1, 0, 0, 1, 0, 0))
    mats = [
        dict(pbrBaseColorFactor=[0.35, 0.1, 0.4, 1], pbrRoughnessFactor=0.8, pbrMetallicFactor=0.0, sheenColorFactor=[0.9, 0.8, 1.0], sheenRoughnessFactor=0.6,
             sheenColorTexture=ti(noise_rgba(True)), sheenRoughnessTexture=ti(noise_rgba())),
        dict(pbrBaseColorFactor=[0.9, 0.9, 0.9, 1], pbrRoughnessFactor=0.3, pbrMetallicFactor=1.0, iridescenceFactor=1.0, iridescenceIor=1.35,
             iridescenceThicknessMinimum=150.0, iridescenceThicknessMaximum=650.0, iridescenceTexture=ti(noise_rgba(lo=0.5)),
             iridescenceThicknessTexture=ti(noise_rgba(), 1)),
        dict(pbrBaseColorFactor=[0.8, 0.6, 0.3, 1], pbrRoughnessFactor=0.35, pbrMetallicFactor=1.0, anisotropyStrength=0.8,
             anisotropyRotation=[math.sin(0.6), math.cos(0.6)], anisotropyTexture=ti(noise_rgba(lo=0.2), transform=True)),
        dict(pbrBaseColorFactor=[0.2, 0.5, 0.3, 1], pbrRoughnessFactor=0.4, pbrMetallicFactor=0.0, specularFactor=0.8, specularColorFactor=[1.0, 0.7, 0.5],
             specularTexture=ti(noise_rgba(lo=0.4)), specularColorTexture=ti(noise_rgba(True, lo=0.4)), pbrBaseColorTexture=ti(t_base),
             pbrMetallicRoughnessTexture=ti(t_mr), normalTexture=ti(t_nm), normalTextureScale=0.8),
        dict(pbrBaseColorFactor=[0.7, 0.1, 0.1, 1], pbrRoughnessFactor=0.5, pbrMetallicFactor=0.0, clearcoatFactor=0.9, clearcoatRoughness=0.3,
             clearcoatTexture=ti(noise_rgba(lo=0.5)), clearcoatRoughnessTexture=ti(noise_rgba()), clearcoatNormalTexture=ti(t_nm)),
        dict(pbrBaseColorFactor=[0.9, 0.95, 1.0, 1], pbrRoughnessFactor=0.1, pbrMetallicFactor=0.0, transmissionFactor=0.95, ior=1.45, thicknessFactor=0.8,
             attenuationColor=[0.6, 0.85, 0.7], attenuationDistance=0.7, transmissionTexture=ti(noise_rgba(lo=0.6)), thicknessTexture=ti(noise_rgba(lo=0.5))),
        dict(pbrBaseColorFactor=[0.8, 0.8, 0.3, 1], pbrRoughnessFactor=0.7, pbrMetallicFactor=0.0, diffuseTransmissionFactor=0.7,
             diffuseTransmissionColor=[0.9, 0.6, 0.4], diffuseTransmissionTexture=ti(noise_rgba(lo=0.5)), diffuseTransmissionColorTexture=ti(noise_rgba(True, lo=0.4)),
             doubleSided=1),
        dict(pbrModel=1, pbrDiffuseFactor=[0.7, 0.5, 0.4, 1], pbrSpecularFactor=[0.6, 0.6, 0.6], pbrGlossinessFactor=0.8,
             pbrDiffuseTexture=ti(noise_rgba(True, lo=0.3, alpha=1.0)), pbrSpecularGlossinessTexture=ti(noise_rgba(True, lo=0.0, hi=0.9))),
        dict(pbrBaseColorFactor=[0.2, 0.2, 0.2, 1], pbrRoughnessFactor=0.6, pbrMetallicFactor=0.0, emissiveFactor=[2.0, 1.2, 0.4], emissiveTexture=ti(noise_rgba(True, lo=0.0))),
        dict(pbrBaseColorFactor=[0.3, 0.6, 0.9, 0.6], pbrRoughnessFactor=0.5, pbrMetallicFactor=0.0, alphaMode=2, doubleSided=1, pbrBaseColorTexture=ti(noise_rgba(True, lo=0.3))),
    ]
    ids = [scn.add_material(**m) for m in mats]
    for k, m in enumerate(ids):
        pos, nrm, uv, tan, idx = _sphere(-2.4 + 1.2 * (k % 5), 0.55 + 1.25 * (k // 5), -0.3 * (k // 5), 0.5, n=20)
        uv1 = uv[:, ::-1] * 0.7 + 0.1
        col = None
        if k == 0:  # vertex colours (COLOR_0 as packed unorm4x8)
            c = _u8(np.concatenate([0.6 + 0.4 * rng.random((len(pos), 3)), np.ones((len(pos), 1))], 1)).astype(np.uint32)
            col = c[:, 0] | (c[:, 1] << 8) | (c[:, 2] << 16) | (c[:, 3] << 24)
        scn.add_node(scn.add_primitive(pos, idx, normals=nrm, uv0=uv, uv1=uv1, tangents=tan, colors=col), m)

    def ground(u, v):
        return _xyz((u * 2 - 1) * 6, np.zeros_like(u), (1 - v * 2) * 6)
    gm = scn.add_material(pbrBaseColorFactor=[0.6, 0.6, 0.6, 1], pbrRoughnessFactor=0.8, pbrMetallicFactor=0.0, pbrBaseColorTexture=ti(t_base, transform=True))
    scn.add_node(scn.add_primitive(*_split(param_surface(ground, 6, 6, (3, 3)))), gm)
    cam = Camera()
    cam.eye = np.array([0.0, 1.6, 5.6], np.float32)
    cam.center = np.array([0.0, 1.1, 0.0], np.float32)
    cam.yfov = math.radians(45.0)
    cam.znear, cam.zfar = 0.05, 100.0
    scn.camera = cam
    return scn


def synth_animated(seed=1234, tex_size=64):
    """Deforming geometry for the animation feed (b200pt_set_animation / b200pt_animate; shaders/skinning.comp.slang,
    shaders/morph.comp.slang): a normal-mapped ground, a SKINNED tube (3 joints, blended weights, unused influence slots with
    weight 0 / joint -1 / a joint index beyond the skin) instanced twice (one instance mirrored), a MORPHED sphere (2 targets with
    position, normal and tangent deltas) and a banner that is BOTH morphed and skinned (morph -> skin composition,
    src/gltf_scene_animation_vk.cpp:545-556).  Returns (scene, morph_tasks, skin_tasks, pose) with pose(k) -> (morph weights per
    morph task, joint matrices per skin task, normal matrices per skin task) for a few key poses."""
    from .animation import MorphTask, SkinTask, joint_matrices
    rng = np.random.default_rng(seed)
    scn = Scene()
    base, mr, nm = make_texture_set(tex_size, rng, (0.7, 0.72, 0.68))
    tb, tm, tn = scn.add_texture(base, srgb=True), scn.add_texture(mr), scn.add_texture(nm)
    textured = dict(pbrBaseColorTexture=scn.add_texture_info(tb), pbrMetallicRoughnessTexture=scn.add_texture_info(tm),
                    normalTexture=scn.add_texture_info(tn))
    m_floor = scn.add_material(pbrBaseColorFactor=[1, 1, 1, 1], pbrRoughnessFactor=1.0, pbrMetallicFactor=0.1, **textured)
    m_arm = scn.add_material(pbrBaseColorFactor=[0.9, 0.55, 0.35, 1], pbrRoughnessFactor=0.6, pbrMetallicFactor=0.0, **textured)
    m_blob = scn.add_material(pbrBaseColorFactor=[0.85, 0.85, 0.9, 1], pbrRoughnessFactor=0.3, pbrMetallicFactor=1.0, **textured)
    m_flag = scn.add_material(pbrBaseColorFactor=[0.3, 0.5, 0.85, 1], pbrRoughnessFactor=0.7, pbrMetallicFactor=0.0, doubleSided=1, **textured)

    def ground(u, v):
        return _xyz((u * 2 - 1) * 5, np.zeros_like(u), (1 - v * 2) * 5)
    scn.add_node(scn.add_primitive(*_split(param_surface(ground, 6, 6, (3, 3)))), m_floor)

    # --- skinned tube: object space along +y, 0..2.4 ---
    def tube(u, v):
        a = u * 2 * math.pi
        return _xyz(0.25 * np.cos(a), v * 2.4, -0.25 * np.sin(a))
    tp = _split(param_surface(tube, 20, 24, (2, 4)))
    arm = scn.add_primitive(*tp)
    pos = tp[0]
    y = pos[:, 1] / 2.4
    w = np.zeros((len(pos), 4), np.float32)
    j = np.zeros((len(pos), 4), np.int32)
    w[:, 0] = np.clip(1.0 - y * 2.0, 0, 1)
    w[:, 2] = np.clip(y * 2.0 - 1.0, 0, 1)
    w[:, 1] = 1.0 - w[:, 0] - w[:, 2]
    j[:, 0], j[:, 1], j[:, 2] = 0, 1, 2
    j[:, 3] = np.where(np.arange(len(pos)) % 3 == 0, -1, 7)   # unused slot: weight 0 with a negative / out-of-range joint
    w[::5, 3] = 0.25                                           # ... and a positive weight on an out-of-range joint (skipped by the shader)
    j[::5, 3] = 7
    arm_t = np.eye(4)
    arm_t[:3, 3] = [-1.8, 0.0, 0.3]
    scn.add_node(arm, m_arm, arm_t)
    arm_m = np.diag([-1.0, 1.0, 1.0, 1.0])
    arm_m[:3, 3] = [2.4, 0.0, -0.8]
    scn.add_node(arm, m_arm, arm_m)
    skin_arm = SkinTask(arm, pos.copy(), w, j, 3, base_normals=tp[2].copy(), base_tangents=tp[5].copy())

    # --- morphed sphere ---
    sp = _split(_sphere(0.0, 1.0, 0.0, 0.7, n=28))
    blob = scn.add_primitive(*sp)
    bp, bn, bt = sp[0], sp[2], sp[5]
    d0 = (bn * (0.35 * np.maximum(0.0, np.sin(6.0 * bp[:, 1:2])))).astype(np.float32)              # ribs along the normal
    d1 = np.stack([0.4 * (bp[:, 1] - 1.0) * bp[:, 2], np.zeros(len(bp)), -0.4 * (bp[:, 1] - 1.0) * bp[:, 0]], 1).astype(np.float32)  # twist
    dn = (rng.normal(size=(2, len(bp), 3)) * 0.15).astype(np.float32)
    dt = (rng.normal(size=(2, len(bp), 3)) * 0.10).astype(np.float32)
    blob_t = np.eye(4)
    blob_t[:3, 3] = [0.2, 0.0, -0.4]
    scn.add_node(blob, m_blob, blob_t)
    morph_blob = MorphTask(blob, bp.copy(), np.stack([d0, d1]), base_normals=bn.copy(), base_tangents=bt.copy(), normal_deltas=dn, tangent_deltas=dt)

    # --- banner: morphed (wave) and then skinned (2 joints) ---
    def banner(u, v):
        return _xyz(u * 1.6, v * 1.0, np.zeros_like(u))
    fp = _split(param_surface(banner, 16, 10, (2, 1)))
    flag = scn.add_primitive(*fp)
    fpos = fp[0]
    wave = np.stack([np.zeros(len(fpos)), np.zeros(len(fpos)), 0.2 * np.sin(5.0 * fpos[:, 0])], 1).astype(np.float32)
    fw = np.zeros((len(fpos), 4), np.float32)
    fj = np.zeros((len(fpos), 4), np.int32)
    fw[:, 1] = np.clip(fpos[:, 0] / 1.6, 0, 1)
    fw[:, 0] = 1.0 - fw[:, 1]
    fj[:, 1] = 1
    flag_t = np.eye(4)
    flag_t[:3, 3] = [0.9, 1.3, 1.0]
    scn.add_node(flag, m_flag, flag_t)
    morph_flag = MorphTask(flag, fpos.copy(), wave[None], base_normals=fp[2].copy(), base_tangents=fp[5].copy())
    skin_flag = SkinTask(flag, fpos.copy(), fw, fj, 2, base_normals=fp[2].copy(), base_tangents=fp[5].copy())

    scn.lights = [_light("point", position=(0.5, 3.5, 2.5), color=(1.0, 0.95, 0.9), intensity=25.0)]
    cam = Camera()
    cam.eye = np.array([0.4, 2.4, 5.6], np.float32)
    cam.center = np.array([0.1, 1.0, 0.0], np.float32)
    cam.yfov = math.radians(45.0)
    cam.znear, cam.zfar = 0.05, 100.0
    scn.camera = cam

    def rot_z(a, pivot_y):
        c, s_ = math.cos(a), math.sin(a)
        r = np.array([[c, -s_, 0, 0], [s_, c, 0, 0], [0, 0, 1, 0], [0, 0, 0, 1.0]])
        t0, t1 = np.eye(4), np.eye(4)
        t0[1, 3], t1[1, 3] = -pivot_y, pivot_y
        return t1 @ r @ t0

    def pose(k):
        a = [0.0, 0.45, -0.7][k % 3]
        # the arm's skeleton: joint nodes at y = 0 / 0.8 / 1.6 in the mesh node's frame, a chain bending about z; bind = rest pose
        rest = [np.eye(4) for _ in range(3)]
        for i, yy in enumerate((0.0, 0.8, 1.6)):
            rest[i][1, 3] = yy
        b1, b2 = rot_z(a, 0.8), rot_z(a, 0.8) @ rot_z(1.3 * a, 1.6)
        world = [np.eye(4), rest[0], b1 @ rest[1], b2 @ rest[2]]           # node 0 = mesh node, 1..3 = joints
        jm_arm, nm_arm = joint_matrices(world, [1, 2, 3], [np.linalg.inv(r) for r in rest], 0)
        sc = np.diag([1.0, 1.0 + 0.3 * a, 1.0, 1.0])
        fworld = [np.eye(4), np.eye(4), rot_z(0.8 * a, 0.5) @ sc]
        jm_flag, nm_flag = joint_matrices(fworld, [1, 2], [np.eye(4)], 0)   # fewer inverse-bind matrices than joints: identity (:201-205)
        mw = [np.array([[0.0, 0.0], [0.8, -0.5], [0.3, 1.0]][k % 3], np.float32), np.array([[0.0], [1.0], [-0.6]][k % 3], np.float32)]
        return mw, [jm_arm, jm_flag], [nm_arm, nm_flag]
    return scn, [morph_blob, morph_flag], [skin_arm, skin_flag], pose


def synth_hierarchy(seed=1234):
    """A scene graph for the device-side rigid feed (b200pt_set_node_hierarchy / b200pt_update_node_matrices;
    shaders/world_matrix_propagate.comp.slang, update_render_instances.comp.slang): the lit test scene's four render nodes hang
    in a four-level hierarchy (root -> turntable -> arm -> hand, plus a sibling chain listed child-before-parent so that the BFS
    order is not the index order), one render node carries an instance matrix.  Returns (scene, parents, mappings, inst_local,
    pose) with pose(k) -> local matrices [numNodes, 4, 4] (mathematical)."""
    scn = synth_lit(seed)
    #           0 root  1 turntable  2 arm  3 hand  4 leaf-of-5  5 under root   6 unused
    parents = [-1, 0, 1, 2, 5, 0, -1]
    # render nodes: ground, sphere 0, 1, 2  ->  graph nodes
    graph_of = [0, 3, 4, 2]
    mappings = [(graph_of[i], rn["materialID"], rn["renderPrimID"]) for i, rn in enumerate(scn.render_nodes)]
    inst = np.stack([np.eye(4)] * len(scn.render_nodes))
    inst[2] = np.array([[0.9, 0, 0.1, 0.2], [0, 1.1, 0, 0.1], [-0.1, 0, 0.9, -0.3], [0, 0, 0, 1.0]])

    def pose(k):
        a = [0.0, 0.6, -1.1][k % 3]
        c, s_ = math.cos(a), math.sin(a)
        ry = np.array([[c, 0, s_, 0], [0, 1, 0, 0], [-s_, 0, c, 0], [0, 0, 0, 1.0]])
        def tr(x, y, z):
            m = np.eye(4)
            m[:3, 3] = [x, y, z]
            return m
        loc = [np.eye(4), ry @ tr(0.2 * k, 0, 0), tr(0.5, 0.1 * k, 0) @ np.diag([1.0, 1.0 + 0.2 * k, 1.0, 1.0]), tr(-0.3, 0.2, 0.4) @ ry,
               np.diag([-1.0, 1.0, 1.0, 1.0]) @ tr(0.3 * k, 0, 0), tr(0, 0.15 * k, -0.5) @ ry.T, tr(9, 9, 9)]
        return np.asarray(loc, np.float64)
    return scn, np.asarray(parents, np.int32), mappings, inst, pose


def triangle_soup(n, seed=1234, extent=1.0, size=0.15, vertices=None, double_sided=0, material=None):
    """n random triangles in a cube: stress input for traversal parity tests.  vertices: (n, 3, 3) triangles to use instead;
    material: add_material arguments that replace the default ones (e.g. an alpha mode)."""
    if vertices is None:
        rng = np.random.default_rng(seed)
        c = (rng.random((n, 1, 3)) - 0.5) * 2 * extent
        v = c + (rng.random((n, 3, 3)) - 0.5) * 2 * size
    else:
        v = np.asarray(vertices, np.float32)
        n = len(v)
    scn = Scene()
    m = scn.add_material(**dict(dict(pbrBaseColorFactor=[0.8, 0.8, 0.8, 1], pbrMetallicFactor=0.0, doubleSided=double_sided), **(material or {})))
    p = scn.add_primitive(v.reshape(-1, 3), np.arange(n * 3).reshape(-1, 3))
    scn.add_node(p, m)
    return scn


def icosahedron(radius=1.0):
    """The 12 vertices (float64 [12, 3]) and 20 faces (int [20, 3], counter-clockwise seen from outside) of a regular
    icosahedron with circumradius `radius` centred on the origin."""
    g = (1.0 + math.sqrt(5.0)) / 2.0
    v = np.array([[-1, g, 0], [1, g, 0], [-1, -g, 0], [1, -g, 0], [0, -1, g], [0, 1, g], [0, -1, -g], [0, 1, -g],
                  [g, 0, -1], [g, 0, 1], [-g, 0, -1], [-g, 0, 1]], np.float64)
    v *= radius / np.linalg.norm(v[0])
    f = np.array([[0, 11, 5], [0, 5, 1], [0, 1, 7], [0, 7, 10], [0, 10, 11], [1, 5, 9], [5, 11, 4], [11, 10, 2], [10, 7, 6],
                  [7, 1, 8], [3, 9, 4], [3, 4, 2], [3, 2, 6], [3, 6, 8], [3, 8, 9], [4, 9, 5], [2, 4, 11], [6, 2, 10],
                  [8, 6, 7], [9, 8, 1]])
    return v, f


def synth_furnace_polyhedron(materials, view=(0.31, 0.52, 1.0), radius=1.0):
    """A convex icosahedron seen by an orthographic camera, for tests of the estimator's expectation.  Each of the 20 faces
    is its own render node (node k = face k, object id k + 1) with three unshared vertices that carry the flat face normal,
    so the shading normal is the geometric one.  `materials` is a list of add_material keyword dicts, given to the faces in
    turn.  The orthographic camera looks along -`view`, so every pixel of a face sees it from the same direction; the body is
    convex, so every ray leaving a face escapes to the environment and no shadow ray from a face is blocked by the body.
    Returns (scene, face normals float64 [20, 3])."""
    v, f = icosahedron(radius)
    scn = Scene()
    mats = [scn.add_material(**m) for m in materials]
    normals = np.empty((20, 3))
    for k, tri in enumerate(f):
        p = v[tri]
        n = np.cross(p[1] - p[0], p[2] - p[0])
        n /= np.linalg.norm(n)
        normals[k] = n
        prim = scn.add_primitive(p, np.array([[0, 1, 2]]), normals=np.repeat(n[None], 3, 0))
        scn.add_node(prim, mats[k % len(mats)])
    cam = Camera()
    cam.type = "orthographic"
    d = np.asarray(view, np.float64) / np.linalg.norm(view)
    cam.eye = (d * 4.0 * radius).astype(np.float32)
    cam.center = np.zeros(3, np.float32)
    cam.xmag = cam.ymag = 1.05 * radius
    cam.znear, cam.zfar = 0.1 * radius, 10.0 * radius
    scn.camera = cam
    return scn, normals


def synth_enclosure(rho, emission, half=1.0):
    """A closed cube of side 2 * `half` whose six walls face inward: single-sided, emissive (`emission`, RGB) Lambertian
    walls (base colour `rho`, metallic 0, specular 0, so the diffuse lobe is the only lobe) and a perspective camera inside.
    Every path stays inside, so every pixel has the same expected value."""
    scn = Scene()
    rho = [rho] * 3 if np.isscalar(rho) else list(rho)
    m = scn.add_material(pbrBaseColorFactor=rho + [1.0], pbrMetallicFactor=0.0, pbrRoughnessFactor=1.0, specularFactor=0.0,
                         emissiveFactor=list(emission), doubleSided=0)
    pos, nrm, idx = [], [], []
    for axis in range(3):
        for s in (-1.0, 1.0):
            n = np.zeros(3)
            n[axis] = -s                     # inward
            a, b = [(axis + 1) % 3, (axis + 2) % 3]
            quad = []
            for u, w in ((-1, -1), (1, -1), (1, 1), (-1, 1)):
                p = np.zeros(3)
                p[axis], p[a], p[b] = s * half, u * half, w * half
                quad.append(p)
            quad = np.array(quad)
            if np.dot(np.cross(quad[1] - quad[0], quad[2] - quad[0]), n) < 0:
                quad = quad[::-1]
            base = len(pos) * 4
            pos.append(quad)
            nrm.append(np.repeat(n[None], 4, 0))
            idx += [[base, base + 1, base + 2], [base, base + 2, base + 3]]
    scn.add_node(scn.add_primitive(np.concatenate(pos), np.array(idx), normals=np.concatenate(nrm)), m)
    cam = Camera()
    cam.eye = np.array([0.1, -0.2, 0.3], np.float32) * half
    cam.center = np.array([0.6, 0.1, -1.0], np.float32) * half
    cam.yfov = math.radians(70.0)
    cam.znear, cam.zfar = 0.01 * half, 10.0 * half
    scn.camera = cam
    return scn


def synth_medium_box(material, half=(4.0, 4.0, 0.5), view=1.0):
    """An axis-aligned box [-hx, hx] x [-hy, hy] x [-hz, hz] (`half` = (hx, hy, hz)) of one material, for tests of the
    participating-media estimator: one render node, 24 unshared vertices carrying the outward flat normal of their face (so
    the shading normal is the geometric one).  `material` is an add_material keyword dict; give it transmission 1,
    metallic 0 and thicknessFactor > 0 for a medium.  An orthographic camera on +z looks down -z at the +z face over
    [-view, view]^2, so with view < min(hx, hy) every camera ray enters the box at normal incidence through that face."""
    hx, hy, hz = (float(h) for h in half)
    scn = Scene()
    m = scn.add_material(**material)
    pos, nrm, idx = [], [], []
    ext = (hx, hy, hz)
    for axis in range(3):
        for s in (-1.0, 1.0):
            n = np.zeros(3)
            n[axis] = s
            a, b = (axis + 1) % 3, (axis + 2) % 3
            quad = []
            for u, w in ((-1, -1), (1, -1), (1, 1), (-1, 1)):
                p = np.zeros(3)
                p[axis], p[a], p[b] = s * ext[axis], u * ext[a], w * ext[b]
                quad.append(p)
            quad = np.array(quad)
            if np.dot(np.cross(quad[1] - quad[0], quad[2] - quad[0]), n) < 0:
                quad = quad[::-1]
            base = len(pos) * 4
            pos.append(quad)
            nrm.append(np.repeat(n[None], 4, 0))
            idx += [[base, base + 1, base + 2], [base, base + 2, base + 3]]
    scn.add_node(scn.add_primitive(np.concatenate(pos), np.array(idx), normals=np.concatenate(nrm)), m)
    cam = Camera()
    cam.type = "orthographic"
    cam.eye = np.array([0.0, 0.0, hz + 4.0], np.float32)
    cam.center = np.array([0.0, 0.0, 0.0], np.float32)
    cam.up = np.array([0.0, 1.0, 0.0], np.float32)
    cam.xmag = cam.ymag = float(view)
    cam.znear, cam.zfar = 0.1, 2.0 * hz + 8.0
    scn.camera = cam
    return scn


def scene_state(scn):
    """Plain-python snapshot of a Scene (for caching generated workloads)."""
    import ctypes as C
    cam = scn.camera
    return dict(render_nodes=scn.render_nodes, render_prims=scn.render_prims,
                materials=[bytes(m) for m in scn.materials], texture_infos=[bytes(t) for t in scn.texture_infos],
                textures=scn.textures, lights=[bytes(l) for l in scn.lights],
                camera=None if cam is None else dict(cam.__dict__))


def scene_from_state(st):
    from . import abi
    scn = Scene()
    scn.render_nodes, scn.render_prims, scn.textures = st["render_nodes"], st["render_prims"], st["textures"]
    scn.materials = [abi.ShadeMaterial.from_buffer_copy(b) for b in st["materials"]]
    scn.texture_infos = [abi.TextureInfo.from_buffer_copy(b) for b in st["texture_infos"]]
    scn.lights = [abi.Light.from_buffer_copy(b) for b in st["lights"]]
    if st["camera"] is not None:
        scn.camera = Camera()
        scn.camera.__dict__.update(st["camera"])
    return scn
