"""Float64 model of the camera stage: what a pixel of the accumulation image converges to when the scene is made of unlit,
single-triangle regions of constant colour over a backdrop.

The stage restated (processPixel / samplePixel / getRay of the reference's path tracer):
- seed = xxhash32(x, y, frameCount); the first sample of a frame is offset by 0.5 + 0.4246609 (r cos t, r sin t) with
  r = sqrt(-2 ln max(1e-38, u1)), t = 2 pi u2 (on a DLSS frame by 0.5 + the frame's jitter, without the two draws); samples
  s >= 1 by (u, u') uniform on the unit square.  The draws are on a 2^-23 grid: the Gaussian is modelled untruncated, which
  misplaces a mass of about 1.2e-7 (the tail beyond u1 = 2^-23).
- clip = (p + offset) / imageSize * 2 - 1 with the full frame's imageSize and global row; a pinhole ray starts at the eye, an
  orthographic one on the view plane and runs along the view axis.
- Depth of field (perspective only): the lens point is (cos r1 a + sin r1 b) sqrt(r2) with r1 = 2 pi u, r2 = u' aperture, so it is
  uniform on a disk of radius sqrt(aperture); a and b are mul(viewMatrixI, (1,0,0,0)) and mul(viewMatrixI, (0,1,0,0)), which on
  the glm matrices are the first two ROWS of the camera-to-world rotation, not its right and up columns.  The ray starts at
  eye + lens and passes through eye + focalDistance * d, d the unit pinhole direction: the focal surface is a sphere.
- An unlit hit returns its base colour with .w = 1 (solid); a primary miss the background colour (solid background) or the
  environment times envIntensity, with .w = 0.  The firefly clamp scales the whole float4 by threshold / mean(rgb) when
  mean(rgb) > threshold.
- The frame value is the mean of numSamples samples; frames fold into the running mean (old T + c N) / (T + N).

The camera is derived from its parameters (eye, center, up, yfov or xmag / ymag, width / height), never from the frame info's
matrices; rays_from_frame_info restates getRay on those matrices for a self-check.

A pixel's expectation is sum_k p_k c(L_k), p_k the probability that its sample lands in region k:
- pinhole / orthographic: a triangle's preimage in offset space is its projection on the screen.  The Gaussian mass of a polygon
  is a signed sum over its edges of the mass of the triangle (centre, a_i, a_i+1), which is closed-form in Owen's T function;
  the box mass is the area of polygon & unit square.
- thin lens: for a fixed offset o, the central projection from the focal point F(o) maps the triangle onto the lens plane as a
  triangle; the covered fraction A(o) is area(disk & that triangle) / area(disk), closed-form.  A(o) is only piecewise smooth,
  so it is integrated over o with composite Gauss-Legendre rules at two orders that must agree.
"""
import math

import numpy as np
from scipy import special

SIGMA = 0.4246609
# where the Gaussian offset can reach from the pixel's corner: 0.5 + sqrt(-2 ln 1e-38) sigma
GAUSS_REACH = 0.5 + math.sqrt(-2.0 * math.log(1e-38)) * SIGMA


# ---- camera -----------------------------------------------------------------------------------------------------------------
class Cam:
    """the camera of a scene.Camera at a width x height frame, from its parameters, in float64"""

    def __init__(self, cam, width, height):
        self.w, self.h = int(width), int(height)
        self.eye = np.asarray(cam.eye, np.float64)
        f = np.asarray(cam.center, np.float64) - self.eye
        f /= np.linalg.norm(f)
        s = np.cross(f, np.asarray(cam.up, np.float64))
        s /= np.linalg.norm(s)
        u = np.cross(s, f)
        self.R = np.stack([s, u, -f], 1)          # camera to world: columns right, up, back
        self.ortho = cam.type == "orthographic"
        if self.ortho:
            self.sx, self.sy = float(cam.xmag), float(cam.ymag)
            self.z0 = float(cam.zfar) - 2.0 * float(cam.znear)   # view z of clip z = -1 under the [0, 1] orthographic depth
        else:
            t = math.tan(float(cam.yfov) / 2.0)
            self.sx, self.sy = t * self.w / self.h, t
        # the lens basis: the first two rows of the camera-to-world rotation
        self.lens_a, self.lens_b = self.R[0].copy(), self.R[1].copy()

    def ray(self, px, py):
        """screen positions (pixel + offset, global rows) -> origins [n, 3], unit directions [n, 3]"""
        cx = np.asarray(px, np.float64) / self.w * 2.0 - 1.0
        cy = np.asarray(py, np.float64) / self.h * 2.0 - 1.0
        if self.ortho:
            v = np.stack([cx * self.sx, -cy * self.sy, np.full_like(cx, self.z0)], -1)
            return self.eye + v @ self.R.T, np.broadcast_to(-self.R[:, 2], v.shape).copy()
        v = np.stack([cx * self.sx, -cy * self.sy, -np.ones_like(cx)], -1)
        d = v @ self.R.T
        return np.broadcast_to(self.eye, d.shape).copy(), d / np.linalg.norm(d, axis=-1, keepdims=True)

    def view(self, p):
        return (np.asarray(p, np.float64) - self.eye) @ self.R

    def project(self, p):
        """world points [n, 3] -> screen positions [n, 2]; asserts they lie in front of the camera"""
        q = self.view(p)
        if self.ortho:
            cx, cy = q[..., 0] / self.sx, -q[..., 1] / self.sy
        else:
            assert np.all(-q[..., 2] > 1e-6), "a vertex behind the camera"
            cx, cy = q[..., 0] / (-q[..., 2] * self.sx), -q[..., 1] / (-q[..., 2] * self.sy)
        return np.stack([(cx + 1.0) * 0.5 * self.w, (cy + 1.0) * 0.5 * self.h], -1)

    def px_per_unit(self, depth):
        """screen pixels per world unit across the view, at view depth `depth`"""
        return self.h / (2.0 * self.sy * (1.0 if self.ortho else depth))


def rays_from_frame_info(fi, px, py):
    """getRay on the frame info's float32 matrices, evaluated in float64: the self-check of Cam.ray"""
    projI = np.asarray(fi.projInv, np.float64).reshape(4, 4)     # glm bytes: row k of this array is column k of the matrix
    viewI = np.asarray(fi.viewInv, np.float64).reshape(4, 4)
    cx = np.asarray(px, np.float64) / fi.imageSize[0] * 2.0 - 1.0
    cy = np.asarray(py, np.float64) / fi.imageSize[1] * 2.0 - 1.0
    vc = np.stack([cx, cy, -np.ones_like(cx), np.ones_like(cx)], -1) @ projI      # mul(v, M)
    vc = vc / vc[:, 3:]
    if fi.flags & 1:   # SCENE_IS_ORTHOGRAPHIC
        o = (vc @ viewI)[:, :3]
        d = np.broadcast_to((np.array([0.0, 0.0, -1.0, 0.0]) @ viewI)[:3], o.shape)
    else:
        o = np.broadcast_to(viewI[3, :3], vc[:, :3].shape)
        d = (vc @ viewI)[:, :3] - o
    return o.copy(), d / np.linalg.norm(d, axis=-1, keepdims=True)


def lens_basis_from_frame_info(fi):
    """mul(viewMatrixI, (1,0,0,0)) and mul(viewMatrixI, (0,1,0,0)) on the frame info's bytes"""
    m = np.asarray(fi.viewInv, np.float64)
    return m[[0, 4, 8]], m[[1, 5, 9]]


# ---- Gaussian and box masses of polygons ------------------------------------------------------------------------------------
def _cross(a, b):
    return a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]


def gauss_tri_mass(A, B):
    """signed mass of the standard 2D normal over the triangle (0, A, B): A, B [..., 2] in units of sigma.  With h the
    distance from 0 to the line AB and a < b the positions of A and B along it, the unsigned mass is
    W(h, atan(b / h)) - W(h, atan(a / h)), W(h, t) = t / 2 pi - T(h, tan t) (Owen's T)"""
    A, B = np.asarray(A, np.float64), np.asarray(B, np.float64)
    e = B - A
    L = np.linalg.norm(e, axis=-1)
    cr = _cross(A, B)
    ok = (L > 0) & (np.abs(cr) > 0)
    Ls = np.where(ok, L, 1.0)
    h = np.where(ok, np.abs(cr) / Ls, 1.0)
    a = np.sum(A * e, -1) / Ls
    b = np.sum(B * e, -1) / Ls

    def W(x):
        return np.arctan(x / h) / (2.0 * math.pi) - special.owens_t(h, x / h)

    return np.where(ok, np.sign(cr) * (W(b) - W(a)), 0.0)


def gauss_poly_mass(poly, center, sigma=SIGMA):
    """mass of N(center, sigma^2 I) over the polygon(s) poly [..., n, 2] (any orientation, simple)"""
    P = (np.asarray(poly, np.float64) - np.asarray(center, np.float64)[..., None, :]) / sigma
    return np.abs(np.sum(gauss_tri_mass(P, np.roll(P, -1, axis=-2)), -1))


def clip_poly(poly, x0, y0, x1, y1):
    """Sutherland-Hodgman clip of one polygon [n, 2] to the box [x0, x1] x [y0, y1]"""
    pts = [tuple(p) for p in np.asarray(poly, np.float64)]
    for axis, lim, keep_less in ((0, x0, False), (0, x1, True), (1, y0, False), (1, y1, True)):
        inside = (lambda p: p[axis] <= lim) if keep_less else (lambda p: p[axis] >= lim)
        out = []
        for i, p in enumerate(pts):
            q = pts[i - 1]
            if inside(p):
                if not inside(q):
                    out.append(_cut(q, p, axis, lim))
                out.append(p)
            elif inside(q):
                out.append(_cut(q, p, axis, lim))
        pts = out
        if not pts:
            break
    return np.array(pts).reshape(-1, 2)


def _cut(q, p, axis, lim):
    t = (lim - q[axis]) / (p[axis] - q[axis])
    return (q[0] + t * (p[0] - q[0]), q[1] + t * (p[1] - q[1]))


def poly_area(poly):
    P = np.asarray(poly, np.float64)
    return 0.5 * abs(np.sum(_cross(P, np.roll(P, -1, axis=0)))) if len(P) >= 3 else 0.0


def box_mass(poly, x, y):
    """area of polygon & [x, x + 1] x [y, y + 1]"""
    return poly_area(clip_poly(poly, x, y, x + 1.0, y + 1.0))


# ---- disk & polygon ---------------------------------------------------------------------------------------------------------
def _disk_seg(A, B, R):
    """signed area of disk(0, R) & triangle (0, A, B), A, B [..., 2]: the parts of AB inside the disk contribute triangles,
    the parts outside circular sectors"""
    d = B - A
    a = np.maximum(np.sum(d * d, -1), 1e-300)
    b = np.sum(A * d, -1)
    c = np.sum(A * A, -1) - R * R
    disc = b * b - a * c
    s = np.sqrt(np.maximum(disc, 0.0))
    t1 = np.clip((-b - s) / a, 0.0, 1.0)
    t2 = np.clip((-b + s) / a, 0.0, 1.0)
    t2 = np.where(disc > 0, t2, t1)
    P1 = A + t1[..., None] * d
    P2 = A + t2[..., None] * d

    def sector(P, Q):
        return 0.5 * R * R * np.arctan2(_cross(P, Q), np.sum(P * Q, -1))

    return sector(A, P1) + 0.5 * _cross(P1, P2) + sector(P2, B)


def disk_poly_area(poly, R):
    """area of disk(0, R) & the polygon(s) poly [..., n, 2]"""
    P = np.asarray(poly, np.float64)
    return np.abs(np.sum(_disk_seg(P, np.roll(P, -1, axis=-2), R), -1))


def lens_preimage(cam, tri, F):
    """the lens-plane triangle [n, 3, 2] (coordinates along the lens basis a, b) whose points l send the ray from eye + l
    through the focal points F [n, 3] into the world triangle tri [3, 3], and s [n, 3] (the central-projection factors of the
    vertices: all > 1 or all < 0 keeps the map free of a pole and every hit in front of the lens)"""
    n = np.cross(cam.lens_a, cam.lens_b)
    V = np.asarray(tri, np.float64)[None, :, :] - F[:, None, :]          # [n, 3, 3]
    s = -((F - cam.eye) @ n)[:, None] / (V @ n)
    P = F[:, None, :] + s[..., None] * V - cam.eye
    return np.stack([P @ cam.lens_a, P @ cam.lens_b], -1), s


def lens_fraction(cam, tri, F, R):
    """the fraction of the lens disk of radius R whose rays through F [n, 3] hit the triangle"""
    Q, s = lens_preimage(cam, tri, F)
    assert np.all((s.min(1) > 1.0 + 1e-9) | (s.max(1) < -1e-9)), "the lens map of a triangle has a pole or a hit behind the lens"
    return disk_poly_area(Q, R) / (math.pi * R * R)


# ---- quadrature -------------------------------------------------------------------------------------------------------------
def composite_gl(lo, hi, cells, q):
    """nodes and weights of a composite Gauss-Legendre rule with `cells` cells of q nodes on [lo, hi]"""
    x, w = np.polynomial.legendre.leggauss(q)
    edges = np.linspace(lo, hi, cells + 1)
    half = 0.5 * (edges[1:] - edges[:-1])
    mid = 0.5 * (edges[1:] + edges[:-1])
    return (mid[:, None] + half[:, None] * x).ravel(), (half[:, None] * w).ravel()


GAUSS_SPAN = 6.5   # the Gaussian rule covers +-6.5 sigma per axis (the mass outside is 1.6e-10)
ORDERS = ((10, 4), (14, 4))         # (cells, nodes per cell) per axis: the low and the high order of the Gaussian rule
BOX_ORDERS = ((4, 4), (6, 4))      # the same for the unit square


def gauss_rule(cells, q):
    g, w = composite_gl(-GAUSS_SPAN, GAUSS_SPAN, cells, q)
    w = w * np.exp(-0.5 * g * g) / math.sqrt(2.0 * math.pi)
    G1, G2 = np.meshgrid(g, g, indexing="ij")
    return np.stack([G1.ravel(), G2.ravel()], -1) * SIGMA + 0.5, np.outer(w, w).ravel()


def box_rule(cells, q):
    g, w = composite_gl(0.0, 1.0, cells, q)
    G1, G2 = np.meshgrid(g, g, indexing="ij")
    return np.stack([G1.ravel(), G2.ravel()], -1), np.outer(w, w).ravel()


# ---- scene model ------------------------------------------------------------------------------------------------------------
def clamp4(rgbw, threshold):
    """the firefly clamp on float4 values [..., 4]: all four channels scaled by threshold / mean(rgb) above the threshold"""
    v = np.asarray(rgbw, np.float64)
    lum = v[..., :3].mean(-1, keepdims=True)
    return np.where(lum > threshold, v * (threshold / np.where(lum > 0, lum, 1.0)), v)


def point_in_tri(p, tri2):
    """p [n, 2] strictly inside the screen triangle tri2 [3, 2] (either orientation)"""
    c = np.stack([_cross(tri2[(i + 1) % 3] - tri2[i], p - tri2[i]) for i in range(3)], -1)
    return np.all(c > 0, -1) | np.all(c < 0, -1)


def seg_dist(p, a, b):
    """distance from points p [n, 2] to the segment ab"""
    d = b - a
    t = np.clip(((p - a) @ d) / (d @ d), 0.0, 1.0)
    return np.linalg.norm(p - a - t[:, None] * d, axis=-1)


class Model:
    """regions: front triangles (world vertices [3, 3], float4 value before the clamp) over a backdrop float4; `aperture` and
    `focal` as in the push constants (aperture 0: no depth of field)"""

    def __init__(self, cam, tris, values, back, threshold, aperture=0.0, focal=1.0):
        self.cam, self.tris = cam, [np.asarray(t, np.float64) for t in tris]
        self.raw = np.asarray(values, np.float64)
        self.raw_all = np.concatenate([self.raw, np.asarray(back, np.float64)[None]])
        self.vals = clamp4(np.concatenate([self.raw, np.asarray(back, np.float64)[None]]), threshold)   # [K + 1, 4]: K = backdrop
        self.lens = aperture > 0 and not cam.ortho
        self.R = math.sqrt(aperture) if self.lens else 0.0
        self.focal = focal
        self.scr = [cam.project(t) for t in self.tris]
        self.blur = [self._blur(t) for t in self.tris]
        self._check_separation()

    def _blur(self, tri):
        """a bound, in pixels, on how far the lens moves a hit on the triangle across the screen"""
        if not self.lens:
            return 0.0
        z = -self.cam.view(tri)[:, 2]
        return float(np.max(self.R * np.abs(1.0 - z / self.focal) * self.cam.px_per_unit(z))) * 1.25 + 0.5

    def _check_separation(self):
        """no ray can hit two front triangles: their screen triangles, grown by their blur, are disjoint"""
        for j in range(len(self.tris)):
            for k in range(j + 1, len(self.tris)):
                a, b = self.scr[j], self.scr[k]
                d = min(min(seg_dist(a, b[i], b[(i + 1) % 3]).min() for i in range(3)),
                        min(seg_dist(b, a[i], a[(i + 1) % 3]).min() for i in range(3)))
                assert not point_in_tri(a, b).any() and not point_in_tri(b, a).any()
                assert d > self.blur[j] + self.blur[k] + 1.0, f"triangles {j} and {k} too close for their blur"

    def edge_dist(self, p):
        """[n, K]: screen distance of points p [n, 2] to each front triangle's outline"""
        return np.stack([np.min([seg_dist(p, s[i], s[(i + 1) % 3]) for i in range(3)], 0) for s in self.scr], -1)

    def region_at(self, p):
        """the region index of the pinhole sample at screen positions p [n, 2] (K = the backdrop)"""
        out = np.full(len(p), len(self.tris))
        for k, s in enumerate(self.scr):
            out[point_in_tri(p, s)] = k
        return out

    def reach(self, box=False):
        """how far from a pixel's centre its samples reach across the screen"""
        r = (math.sqrt(0.5) + 1e-9) if box else GAUSS_REACH + 0.5 * math.sqrt(2.0) - 0.5
        return r + max(self.blur, default=0.0)

    def pixels(self, y0=0, rows=None, row_ids=None):
        """pixel centres [n, 2] of the global rows of a tile"""
        ys = np.arange(y0, y0 + (rows if rows is not None else self.cam.h)) if row_ids is None else np.asarray(row_ids)
        Y, X = np.meshgrid(ys, np.arange(self.cam.w), indexing="ij")
        return np.stack([X.ravel() + 0.5, Y.ravel() + 0.5], -1).astype(np.float64)

    # -- probabilities of one pixel
    def probs(self, x, y, kind, order=1):
        """[K + 1] region probabilities of pixel (x, y) for a sample drawn by kind 'gauss' (the first sample), 'box' (s >= 1) or
        ('point', ox, oy) (a fixed offset: DLSS).  order 0 / 1 picks the low / high quadrature of the lens."""
        K = len(self.tris)
        p = np.zeros(K + 1)
        if isinstance(kind, tuple):
            o = np.array([[x + kind[1], y + kind[2]]])
            if not self.lens:
                p[self.region_at(o)[0]] = 1.0
                return p
            nodes, w = o, np.ones(1)
        elif not self.lens:
            for k, s in enumerate(self.scr):
                p[k] = gauss_poly_mass(s, np.array([x + 0.5, y + 0.5])) if kind == "gauss" else box_mass(s, x, y)
            p[K] = 1.0 - p[:K].sum()
            return p
        else:
            nodes, w = (gauss_rule(*ORDERS[order]) if kind == "gauss" else box_rule(*BOX_ORDERS[order]))
            nodes = nodes + np.array([x, y])
        # thin lens: the pixel's footprint touches at most one triangle (the separation check); integrate its lens fraction
        c = np.array([[x + 0.5, y + 0.5]])
        d = self.edge_dist(c)[0]
        inside = self.region_at(c)[0]
        for k in range(K):
            if d[k] > self.reach() + 1.0:
                p[k] = 1.0 if inside == k else 0.0
                continue
            _, dirs = self.cam.ray(nodes[:, 0], nodes[:, 1])
            F = self.cam.eye + self.focal * dirs
            p[k] = float(np.sum(w * lens_fraction(self.cam, self.tris[k], F, self.R)))
        p[K] = 1.0 - p[:K].sum()
        return p
