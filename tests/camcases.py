"""Scenes, cases and statistics shared by test_camera_expectation.py (the CPU oracle) and test_gpu_camera_expectation.py (the
device): rendered images of unlit single-triangle regions against the float64 camera model of tests/camref.py.

Three unlit triangles with slanted edges lie fronto-parallel to the camera, one nearer than the focal distance, one near it, one
beyond, over a backdrop: a miss (solid background or a constant environment) or one large unlit triangle behind everything.  A
pixel whose samples all land in one region must equal that region's clamped value; the pixels whose samples straddle an edge
(`mixed`) converge to sum_k p_k c(L_k), with the exact variance of their N-frame mean.  The checks:
1. deterministic pixels equal c(L) in every channel, .w included, within float32 running-mean rounding;
2. the mean of the residuals (value - E) / contrast of the mixed pixels (contrast: the pixel's triangle against the backdrop)
   lies within N_SIGMA sigma (estcases.batch_stats over interleaved batches), and sigma <= 0.2 %; the two sides of the edges
   (pixel centre inside or outside the triangle) apart, each per triangle where every group has 300 pixels, else pooled;
3. sum over mixed pixels of (value - E)^2 / (Var / N) lies within the two-sided p > 1e-4 bounds of chi^2 with one degree of
   freedom per pixel (a mixed pixel's samples reach one triangle and the backdrop only -- pixels that reach two triangles
   are left out -- so its four channels are one indicator);
4. the selection id of frame 0 is the pixel-centre region, except within 1e-4 px of an edge;
5. the NDC depth of frame 0 is the depth of a region the pixel's samples can reach, or 1 on a miss.
"""
import math

import numpy as np
from scipy import stats

import camref
import estcases
from vk_gltf_renderer_b200 import camera as camm
from vk_gltf_renderer_b200.scene import Camera, Scene

N_SIGMA = estcases.N_SIGMA
MAX_REL_SIGMA = 0.002
CHI2_P = 1e-4
ENV_RGB = (0.35, 0.5, 0.65)
BACKGROUND = (0.2, 0.25, 0.3)
# region colours (rgb); the luminances 0.8, 2.0, 5.0 and the backdrop's straddle the clamp threshold of the clamp cases
COLOURS = ((0.9, 0.8, 0.7), (1.5, 2.5, 2.0), (6.0, 4.0, 5.0))
BACK_TRI_RGB = (0.1, 0.3, 0.2)
CLAMP = 1.7
NO_CLAMP = 1.0e30
# the triangles in screen fractions (u right, v down) and view depth in units of the focal distance; irrational offsets keep the
# edge slopes off rational pixel phases
_R2, _R3, _R5 = math.sqrt(2.0), math.sqrt(3.0), math.sqrt(5.0)
TRIS_UV = (
    (((0.06 + 0.01 * _R2, 0.10), (0.33, 0.13 + 0.01 * _R3), (0.14 + 0.01 * _R5, 0.42)), 0.62),
    (((0.55, 0.08 + 0.01 * _R5), (0.93 - 0.01 * _R3, 0.20), (0.66 + 0.01 * _R2, 0.43)), 0.75),
    (((0.22 + 0.01 * _R3, 0.60), (0.78, 0.57 + 0.01 * _R2), (0.43, 0.93 - 0.01 * _R5)), 1.85),
)
BACK_DEPTH = 3.0


def camera(kind):
    """'rot': a perspective camera whose rotation is not symmetric; 'axis': axis-aligned (rows = columns, the control);
    'ortho': orthographic"""
    c = Camera()
    c.up = np.array([0.0, 1.0, 0.0], np.float32)
    c.yfov = math.radians(40.0)
    c.znear, c.zfar = 0.05, 60.0
    if kind == "axis":
        c.eye, c.center = np.array([0.0, 0.0, 4.0], np.float32), np.zeros(3, np.float32)
    else:
        c.eye, c.center = np.array([1.0, 0.5, 3.7], np.float32), np.array([0.2, -0.1, -0.3], np.float32)
    if kind == "ortho":
        c.type = "orthographic"
        c.xmag, c.ymag = 1.6, 1.2
    return c


def focal(cam):
    return float(np.linalg.norm(np.asarray(cam.eye, np.float64) - np.asarray(cam.center, np.float64)))


def _place(cm, uv, z):
    """world points on the plane at view depth z (fronto-parallel) at screen fractions uv"""
    uv = np.asarray(uv, np.float64)
    s = 1.0 if cm.ortho else z
    v = np.stack([(2 * uv[:, 0] - 1) * cm.sx * s, -(2 * uv[:, 1] - 1) * cm.sy * s, np.full(len(uv), -z)], -1)
    return cm.eye + v @ cm.R.T


def build_scene(cam, w, h, back):
    """(Scene, world triangles): three unlit triangles, plus the backdrop triangle when back == 'tri'"""
    cm = camref.Cam(cam, w, h)
    fd = focal(cam)
    tris = [_place(cm, uv, z * fd) for uv, z in TRIS_UV]
    scn = Scene()
    for tri, rgb in zip(tris, COLOURS):
        m = scn.add_material(pbrBaseColorFactor=list(rgb) + [1.0], unlit=1, doubleSided=1)
        scn.add_node(scn.add_primitive(tri, np.array([[0, 1, 2]])), m)
    if back == "tri":
        big = _place(cm, [(-4.0, -4.0), (6.0, -4.0), (0.5, 8.0)], BACK_DEPTH * fd)
        m = scn.add_material(pbrBaseColorFactor=list(BACK_TRI_RGB) + [1.0], unlit=1, doubleSided=1)
        scn.add_node(scn.add_primitive(big, np.array([[0, 1, 2]])), m)
        tris_all = tris + [big]
    else:
        tris_all = tris
    scn.camera = cam
    return scn, tris_all


def env_image():
    return np.broadcast_to(np.asarray(ENV_RGB, np.float32), (16, 32, 3)).copy()


def back_value(back):
    if back == "tri":
        return BACK_TRI_RGB + (1.0,)
    return (BACKGROUND if back == "solid" else ENV_RGB) + (0.0,)


def make_model(cam, w, h, case, tris=None, view_cam=None):
    """the camref.Model of a case (view_cam: the camera of one view of a multi-view render)"""
    if tris is None:
        _, tris = build_scene(cam, w, h, case["back"])
    cm = camref.Cam(view_cam or cam, w, h)
    return camref.Model(cm, tris[:3], [c + (1.0,) for c in COLOURS], back_value(case["back"]), case.get("clamp", NO_CLAMP),
                        aperture=case.get("aperture", 0.0), focal=focal(cam))


def frame_info(cam, w, h, case):
    return camm.make_frame_info(cam, w, h, solid_background=case["back"] == "solid", background=BACKGROUND)


# name -> case.  back: 'solid' / 'env' / 'tri'; aperture (lens radius^2, world units) scaled to the image height by lens_aperture
GAUSS = {f"gauss_{c}_{b}_spp{s}": dict(cam=c, back=b, spp=s) for c in ("rot", "ortho") for b in ("solid", "env") for s in (1, 3)}
# an aperture on the orthographic camera must not blur it
LENS = {f"lens_{c}_spp{s}": dict(cam=c, back="tri", spp=s, lens=True) for c in ("rot", "axis", "ortho") for s in (1, 3)}
CLAMPS = {f"clamp_spp{s}": dict(cam="rot", back="env", spp=s, clamp=CLAMP) for s in (1, 3)}
CASES = {**GAUSS, **LENS, **CLAMPS}


def lens_aperture(h):
    """an aperture that blurs the near triangle by a few pixels at image height h"""
    return 0.03 if h <= 64 else 0.006


def resolve(case, h):
    case = dict(case)
    if case.get("lens"):
        case["aperture"] = lens_aperture(h)
    return case


# the DLSS cases: one frame's jitter (SceneFrameInfo::jitter, pixels), held fixed over the frames of the lens case
DLSS_JITTER = (0.23, -0.31)
DLSS = {"dlss_pinhole": dict(cam="rot", back="env", spp=1), "dlss_lens": dict(cam="rot", back="tri", spp=1, lens=True)}


def dlss_offset(fi):
    """the DLSS frame's sample offset 0.5 + jitter, as the float32 code forms it"""
    return tuple(float(np.float32(0.5) + np.float32(j)) for j in fi.jitter)


def check_dlss_point(model, img, offset, row_ids, label, threshold=NO_CLAMP):
    """a DLSS frame without an aperture is deterministic: every pixel is the clamped value of the region at pixel + offset,
    except within 1e-4 px of an edge"""
    p = model.pixels(row_ids=row_ids) - 0.5 + np.asarray(offset)
    region = model.region_at(p)
    keep = model.edge_dist(p).min(1) > 1e-4
    want = np.stack([clamp_f32(model.raw_all[k], threshold).astype(np.float64) for k in range(len(model.vals))])[region]
    img = img.reshape(-1, 4).astype(np.float64)
    bad = keep & (np.abs(img - want) > 2e-6 * np.maximum(np.abs(want), 1e-2)).any(1)
    if bad.any():
        i = np.nonzero(bad)[0][0]
        return [f"{label}: pixel {divmod(i, model.cam.w)} = {img[i]} != {want[i]} ({bad.sum()} pixels)"]
    return []


def push_constant(cam, h, case, frame, spp, total=None):
    return camm.make_push_constant(cam, h, frame_count=frame, total_samples=frame * spp if total is None else total, num_samples=spp,
                                   max_depth=4, firefly_clamp=case.get("clamp", NO_CLAMP), aperture=case.get("aperture", 0.0))


# ---- expectation of an image ------------------------------------------------------------------------------------------------
class Expectation:
    """per pixel of the rows `row_ids` (global): kind ('det' / 'mixed' / 'skip'), the region index of a deterministic pixel,
    E [4] and the variance [4] of the frames' mean of a mixed one"""

    def __init__(self, model, spp, frames, row_ids, max_mixed=None, dlss_offset=None):
        """dlss_offset: every sample at pixel + dlss_offset (DLSS frames with a fixed jitter; their replaced images are
        averaged in float64, so a deterministic pixel is the clamped value itself, not a float32 running mean)"""
        self.model, self.spp, self.frames = model, spp, frames
        self.running = dlss_offset is None
        w = model.cam.w
        self.row_ids = np.asarray(row_ids)
        centres = model.pixels(row_ids=self.row_ids)
        n = len(centres)
        d = model.edge_dist(centres)
        self.centre_region = model.region_at(centres)
        self.edge_d = d.min(1)
        self.near_tri = d.argmin(1)
        reach = model.reach() + 0.05
        self.kind = np.where(self.edge_d > reach, "det", "band").astype(object)
        self.E = np.zeros((n, 4))
        self.var = np.zeros((n, 4))
        self.order_gap = 0.0
        # a pixel whose samples can reach two triangles is not tested as mixed: a mixed pixel straddles exactly one triangle and
        # the backdrop, so its four channels are affine in one indicator (checks 2 and 3 rely on it)
        two = (d <= reach).sum(1) > 1
        # samples beyond 2 px (4.7 sigma) plus the blur from an edge leave a pixel mixed by less than 1e-5: not worth a lens
        # expectation, and neither deterministic
        far = (self.kind == "band") & (self.edge_d > max(model.blur, default=0.0) + 2.0)
        if model.lens:
            self.kind[far] = "skip"
        self.kind[(self.kind == "band") & two] = "skip"
        band = np.nonzero(self.kind == "band")[0]
        if max_mixed is not None and len(band) > max_mixed:
            keep = band[np.linspace(0, len(band) - 1, max_mixed).round().astype(int)]
            self.kind[np.setdiff1d(band, keep)] = "skip"
            band = keep
        vals = model.vals
        for i in band:
            x, y = centres[i] - 0.5
            if dlss_offset is not None:
                ps, weights = [model.probs(x, y, ("point",) + tuple(dlss_offset))], [1.0]
            else:
                pg, pb = model.probs(x, y, "gauss"), model.probs(x, y, "box") if spp > 1 else None
                if model.lens:
                    lo_g = model.probs(x, y, "gauss", order=0)
                    gap = np.abs(lo_g - pg) @ np.abs(vals)
                    if spp > 1:
                        gap = np.maximum(gap, np.abs(model.probs(x, y, "box", order=0) - pb) @ np.abs(vals))
                    self.order_gap = max(self.order_gap, float(gap.max()))
                ps, weights = ([pg, pb], [1.0, spp - 1.0]) if spp > 1 else ([pg], [1.0])
            m = sum(wt * (p @ vals) for p, wt in zip(ps, weights)) / spp
            v = sum(wt * (p @ vals ** 2 - (p @ vals) ** 2) for p, wt in zip(ps, weights)) / spp ** 2
            self.E[i], self.var[i] = m, v / frames
            # the rarer side of the pixel's two regions, in expected samples over the run: >= 10 keeps its mean near normal
            pmin = min(min(1.0 - p.max(), p.max()) for p in ps)
            if pmin * frames * spp >= 10:
                self.kind[i] = "mixed"
            elif 1.0 - min(p.max() for p in ps) < 1e-12:
                self.kind[i] = "det"
            else:
                self.kind[i] = "skip"
        det = np.nonzero(self.kind == "det")[0]
        self.E[det] = vals[self.centre_region[det]]
        self.shape = (len(self.row_ids), w)


def f32_running_mean(value, spp, frames):
    """the float32 running mean of a pixel whose every sample is `value` (float4): the frame mean of spp samples, folded as
    (old T + c N) / (T + N) over the frames; frame 0 replaces the image"""
    f = np.float32
    v = np.asarray(value, np.float32)
    c = v
    for _ in range(spp - 1):
        c = (c + v).astype(np.float32)
    c = (c / f(spp)).astype(np.float32)
    img = c
    for k in range(1, frames):
        t, n = f(k * spp), f(spp)
        img = ((img * t + c * n) / f(k * spp + spp)).astype(np.float32)
    return img.astype(np.float64)


def clamp_f32(rgbw, threshold):
    """the firefly clamp as the float32 code evaluates it"""
    f = np.float32
    r = np.asarray(rgbw, np.float32)
    lum = f((r[0] + r[1]) + r[2]) * f(1.0 / 3.0)
    return (r * f(f(threshold) / lum)).astype(np.float32) if lum > f(threshold) else r


def group_stats(resid, label, report, fails, batches_max=64):
    """pooled mean of residuals (already divided by their contrast) against N_SIGMA sigma, and sigma <= MAX_REL_SIGMA"""
    if len(resid) < 96:
        fails.append(f"{label}: only {len(resid)} mixed pixels")
        return
    n = len(resid)
    mean, sigma = estcases.batch_stats(resid[:, None], batches=min(batches_max, n // 6))
    mean, sigma = float(mean[0]), float(sigma[0])
    report.append(f"{label}: n={n} mean resid/contrast={mean:.3e} sigma={sigma:.3e} |d|/sigma={abs(mean) / max(sigma, 1e-300):.2f}")
    if abs(mean) > N_SIGMA * sigma + 1e-6:
        fails.append(f"band mean off its expectation: {report[-1]}")
    if sigma > MAX_REL_SIGMA:
        fails.append(f"band too noisy to see a 1 % bias: {report[-1]}")


def check_image(ex, img, label, report, threshold=NO_CLAMP):
    """checks 1-3 on an image [rows, W, 4] of the rows of ex; returns the list of failures"""
    img = img.reshape(-1, 4).astype(np.float64)
    fails = []
    det = np.nonzero(ex.kind == "det")[0]
    vals = ex.model.vals
    want = np.stack([f32_running_mean(clamp_f32(ex.model.raw_all[k], threshold), ex.spp, ex.frames) if ex.running
                     else clamp_f32(ex.model.raw_all[k], threshold).astype(np.float64) for k in range(len(vals))])
    err = np.abs(img[det] - want[ex.centre_region[det]])
    tol = 2e-6 * np.maximum(np.abs(want[ex.centre_region[det]]), 1e-2)
    bad = (err > tol).any(1)
    report.append(f"{label}: {len(det)} deterministic pixels, {bad.sum()} off; max |d| {err.max(initial=0):.3g}")
    if bad.any():
        i = det[np.nonzero(bad)[0][0]]
        fails.append(f"{label}: deterministic pixel {divmod(i, ex.shape[1])} = {img[i]} != {want[ex.centre_region[i]]}")
    # checks 2 and 3 on one channel per pixel, the one of the largest contrast: a mixed pixel straddles one triangle and the
    # backdrop, so its four channels are affine in one indicator
    idx = np.nonzero(ex.kind == "mixed")[0]
    tri = ex.near_tri[idx]
    diff = vals[tri] - vals[-1]
    ch = np.argmax(np.abs(diff), 1)
    contrast = np.abs(diff[np.arange(len(idx)), ch])
    r = img[idx, ch] - ex.E[idx, ch]
    # the two sides of an edge apart (pixel centre inside the triangle or outside it): a wrong filter width biases them in
    # opposite directions, which a pooled mean would cancel
    inside = ex.centre_region[idx] == tri
    K = len(ex.model.tris)
    per_tri = all(np.sum((tri == k) & (inside == side)) >= 300 for k in range(K) for side in (False, True))
    for side in (False, True):
        sel = inside == side
        name = "inside" if side else "outside"
        if per_tri:
            for k in range(K):
                m = sel & (tri == k)
                group_stats(r[m] / contrast[m], f"{label} triangle {k} {name}", report, fails)
        else:
            group_stats(r[sel] / contrast[sel], f"{label} all triangles {name}", report, fails)
    chi2 = float(np.sum(r * r / ex.var[idx, ch]))
    dof = len(idx)
    lo, hi = stats.chi2.ppf(CHI2_P / 2, dof), stats.chi2.isf(CHI2_P / 2, dof)
    report.append(f"{label}: chi2 {chi2:.1f} over {dof} pixels, bounds [{lo:.1f}, {hi:.1f}]")
    if not lo <= chi2 <= hi:
        fails.append(f"{label}: chi2 {chi2:.1f} outside [{lo:.1f}, {hi:.1f}] over {dof} mixed pixels")
    return fails


def check_selection(ex, ids, label, n_front=3, back_id=0):
    """check 4: the frame-0 object id is the pixel-centre region's (node + 1), except within 1e-4 px of an edge"""
    ids = ids.reshape(-1)
    want = np.where(ex.centre_region < n_front, ex.centre_region + 1, back_id)
    ok = (ex.edge_d < 1e-4) | (ids == want)
    if not ok.all():
        i = np.nonzero(~ok)[0][0]
        return [f"{label}: selection id {ids[i]} != {want[i]} at pixel {divmod(i, ex.shape[1])} ({(~ok).sum()} pixels)"]
    return []


def ndc_of_depth(cam, z):
    if cam.type == "orthographic":
        return (z - cam.znear) / (cam.zfar - cam.znear)
    return cam.zfar * (z - cam.znear) / ((cam.zfar - cam.znear) * z)


def check_depth(ex, depth, cam, case, label):
    """check 5: a pixel reads the NDC depth of a region its samples can reach, or 1 for a miss"""
    fd = focal(cam)
    zs = [ndc_of_depth(cam, z * fd) for _, z in TRIS_UV]
    zb = ndc_of_depth(cam, BACK_DEPTH * fd) if case["back"] == "tri" else 1.0
    d = depth.reshape(-1).astype(np.float64)
    model = ex.model
    centres = model.pixels(row_ids=ex.row_ids)
    dist = model.edge_dist(centres)
    reach = model.reach() + 0.05
    ok = np.zeros(len(d), bool)
    for k in range(3):
        can = (ex.centre_region == k) | (dist[:, k] <= reach)
        ok |= can & (np.abs(d - zs[k]) <= 2e-6)
    can_back = (ex.centre_region == 3) | (dist.min(1) <= reach)
    ok |= can_back & (np.abs(d - zb) <= 2e-6)
    if not ok.all():
        i = np.nonzero(~ok)[0][0]
        return [f"{label}: NDC depth {d[i]} at pixel {divmod(i, ex.shape[1])} is no reachable region's ({zs}, back {zb}); "
                f"{(~ok).sum()} pixels"]
    return []
