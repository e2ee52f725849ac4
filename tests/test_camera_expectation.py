"""The camera stage against the float64 model of tests/camref.py: the model's own checks, then the CPU oracle's images of the
cases of tests/camcases.py (Gaussian pixel filter, box jitter of later samples, thin lens, firefly clamp, a row tile, the
selection ray and the NDC depth of frame 0).  The device runs the same cases in test_gpu_camera_expectation.py."""
import math

import numpy as np
import pytest
from scipy import special

import camcases as CC
import camref
from vk_gltf_renderer_b200 import abi

W, H = 64, 48
FRAMES = 600
LENS_FRAMES = 1800
# every edge pixel of the lens cases (the device file takes a subset)
LENS_PIXELS = None
# the two quadrature orders of the lens model agree to this fraction of the largest region value, well under the 0.2 % a band
# check resolves
ORDER_TOL = 5e-4


# ---- the model's own checks -------------------------------------------------------------------------------------------------
def test_gauss_mass_half_plane_and_grid():
    rng = np.random.default_rng(1)
    # a triangle far larger than sigma, one edge at distance d from the centre: the mass is the half-plane's erf
    for d in (-0.7, -0.1, 0.0, 0.05, 0.3, 1.1):
        poly = np.array([[-500.0, d], [500.0, d], [0.0, 1000.0]])
        want = 0.5 * special.erfc(d / (camref.SIGMA * math.sqrt(2.0)))
        assert abs(camref.gauss_poly_mass(poly, np.zeros(2)) - want) < 1e-12
    # small random triangles against a dense midpoint grid
    g = np.linspace(-4, 4, 4001)
    step = g[1] - g[0]
    X, Y = np.meshgrid(g, g)
    dens = np.exp(-(X * X + Y * Y) / (2 * camref.SIGMA ** 2)) / (2 * math.pi * camref.SIGMA ** 2) * step * step
    for _ in range(4):
        tri = rng.uniform(-1.5, 1.5, (3, 2))
        inside = camref.point_in_tri(np.stack([X.ravel(), Y.ravel()], -1), tri).reshape(X.shape)
        assert abs(camref.gauss_poly_mass(tri, np.zeros(2)) - dens[inside].sum()) < 2e-4


def test_box_mass():
    tri = np.array([[0.2, 0.1], [3.0, 0.4], [0.5, 2.0]])
    pts = np.random.default_rng(2).uniform(0, 1, (400000, 2))
    assert abs(camref.box_mass(tri, 0.0, 0.0) - camref.point_in_tri(pts, tri).mean()) < 4e-3


def _lens_model(kind):
    case = CC.resolve(CC.CASES[f"lens_{kind}_spp1"], H)
    cam = CC.camera(kind)
    _, tris = CC.build_scene(cam, W, H, case["back"])
    return tris, CC.make_model(cam, W, H, case, tris)


@pytest.mark.parametrize("kind", ["rot", "axis"])
def test_rays_from_parameters_match_frame_info(kind):
    cam = CC.camera(kind)
    fi = CC.frame_info(cam, W, H, dict(back="env"))
    cm = camref.Cam(cam, W, H)
    px, py = np.random.default_rng(3).uniform(-3, 70, (2, 500))
    o1, d1 = cm.ray(px, py)
    o2, d2 = camref.rays_from_frame_info(fi, px, py)
    assert np.abs(d1 - d2).max() < 1e-6
    assert np.abs(o1 - o2).max() < 1e-6
    a, b = camref.lens_basis_from_frame_info(fi)
    assert np.abs(a - cm.lens_a).max() < 1e-6 and np.abs(b - cm.lens_b).max() < 1e-6


def test_ortho_rays_match_frame_info():
    cam = CC.camera("ortho")
    fi = CC.frame_info(cam, W, H, dict(back="env"))
    px, py = np.random.default_rng(4).uniform(-3, 70, (2, 500))
    o1, d1 = camref.Cam(cam, W, H).ray(px, py)
    o2, d2 = camref.rays_from_frame_info(fi, px, py)
    assert np.abs(d1 - d2).max() < 1e-6 and np.abs(o1 - o2).max() < 1e-5


def test_lens_preimage_against_point_in_triangle():
    tris, m = _lens_model("rot")
    cm = m.cam
    rng = np.random.default_rng(5)
    g = np.linspace(-m.R, m.R, 161)
    L = np.stack(np.meshgrid(g, g), -1).reshape(-1, 2)
    for k in range(3):
        o = m.scr[k].mean(0) + rng.uniform(-3, 3, 2)
        _, d = cm.ray(o[:1], o[1:])
        F = cm.eye + m.focal * d
        Q, _ = camref.lens_preimage(cm, tris[k], F)
        # brute force: the ray from eye + l through F against the triangle
        org = cm.eye + L[:, :1] * cm.lens_a + L[:, 1:] * cm.lens_b
        dirs = F - org
        t = tris[k]
        n = np.cross(t[1] - t[0], t[2] - t[0])
        s = ((t[0] - org) @ n) / (dirs @ n)
        X = org + s[:, None] * dirs
        bary = [np.cross(t[(i + 1) % 3] - t[i], X - t[i]) @ n for i in range(3)]
        hit = (s > 0) & np.all(np.stack(bary) > 0, 0)
        assert np.array_equal(hit, camref.point_in_tri(L, Q[0])), k


def test_lens_to_pinhole_as_aperture_vanishes():
    cam = CC.camera("rot")
    case = dict(back="tri", aperture=1e-12)
    _, tris = CC.build_scene(cam, W, H, "tri")
    lens = CC.make_model(cam, W, H, case, tris)
    pin = CC.make_model(cam, W, H, dict(back="tri"), tris)
    rng = np.random.default_rng(6)
    for k in range(3):
        for _ in range(20):
            x, y = np.floor(lens.scr[k][rng.integers(3)] + rng.uniform(-2, 2, 2))
            for off in rng.uniform(0, 1, (3, 2)):
                assert np.allclose(lens.probs(x, y, ("point", *off)), pin.probs(x, y, ("point", *off)), rtol=0, atol=1e-9)


def test_lens_fraction_against_monte_carlo():
    tris, m = _lens_model("rot")
    cm = m.cam
    rng = np.random.default_rng(7)
    n = 10_000_000
    r = m.R * np.sqrt(rng.uniform(0, 1, n))
    th = rng.uniform(0, 2 * math.pi, n)
    for k in range(3):
        # an offset on the triangle's blurred edge
        a, b = m.scr[k][0], m.scr[k][1]
        o = 0.5 * (a + b)
        _, d = cm.ray(o[:1], o[1:])
        F = cm.eye + m.focal * d
        A = float(camref.lens_fraction(cm, tris[k], F, m.R)[0])
        Q, _ = camref.lens_preimage(cm, tris[k], F)
        hit = camref.point_in_tri(np.stack([r * np.cos(th), r * np.sin(th)], -1), Q[0])
        assert 0.05 < A < 0.95
        assert abs(hit.mean() - A) < 5 * math.sqrt(A * (1 - A) / n) + 1e-12


# ---- the oracle -------------------------------------------------------------------------------------------------------------
def _oracle_run(O, case, frames, y0=0, rows=H):
    cam = CC.camera(case["cam"])
    scn, tris = CC.build_scene(cam, W, H, case["back"])
    o = O.Oracle()
    o.set_scene(scn)
    o.set_environment(CC.env_image())
    fi = CC.frame_info(cam, W, H, case)
    acc = np.zeros((rows, W, 4), np.float32)
    ids = np.zeros((rows, W), np.uint32)
    depth = np.zeros((rows, W), np.float32)
    for f in range(frames):
        o.render_frame(fi, CC.push_constant(cam, H, case, f, case["spp"]), acc, y0=y0, rows=rows, object_id=ids if f == 0 else None,
                       ndc_depth=depth if f == 0 else None)
    return cam, tris, acc, ids, depth


def _check(case, cam, tris, acc, ids, depth, rows_ids, label):
    model = CC.make_model(cam, W, H, case, tris)
    frames = LENS_FRAMES if case.get("lens") else FRAMES
    ex = CC.Expectation(model, case["spp"], frames, rows_ids, max_mixed=LENS_PIXELS if model.lens else None)
    report = []
    fails = CC.check_image(ex, acc, label, report, case.get("clamp", CC.NO_CLAMP))
    fails += CC.check_selection(ex, ids, label, back_id=4 if case["back"] == "tri" else 0)
    fails += CC.check_depth(ex, depth, cam, case, label)
    report.append(f"{label}: lens quadrature orders differ by {ex.order_gap:.2e} (largest region value {np.abs(model.vals).max():.2f})")
    print("\n".join(report))
    assert ex.order_gap <= ORDER_TOL * np.abs(model.vals).max(), ex.order_gap
    assert not fails, "\n".join(fails)


@pytest.mark.parametrize("name", sorted(CC.CASES))
def test_oracle_camera(oracle_mod, name):
    case = CC.resolve(CC.CASES[name], H)
    cam, tris, acc, ids, depth = _oracle_run(oracle_mod, case, LENS_FRAMES if case.get("lens") else FRAMES)
    _check(case, cam, tris, acc, ids, depth, np.arange(H), name)


def test_oracle_camera_row_tile(oracle_mod):
    """a strip of rows: getRay takes the global row and the full frame's imageSize"""
    case = CC.resolve(CC.CASES["lens_rot_spp1"], H)
    y0, rows = 17, 23
    cam, tris, acc, ids, depth = _oracle_run(oracle_mod, case, LENS_FRAMES, y0, rows)
    _check(case, cam, tris, acc, ids, depth, np.arange(y0, y0 + rows), "tile")


@pytest.mark.parametrize("name", sorted(CC.DLSS))
def test_oracle_camera_dlss(oracle_mod, name):
    """DLSS frames sample at 0.5 + the frame's jitter without the Gaussian draws and replace the image.  Without an aperture
    the image is deterministic; with one, the replaced images of frames at one jitter average to the lens-only expectation."""
    case = CC.resolve(CC.DLSS[name], H)
    cam = CC.camera(case["cam"])
    scn, tris = CC.build_scene(cam, W, H, case["back"])
    o = oracle_mod.Oracle()
    o.set_scene(scn)
    o.set_environment(CC.env_image())
    fi = CC.frame_info(cam, W, H, case)
    fi.jitter[:] = list(CC.DLSS_JITTER)
    frames = LENS_FRAMES if case.get("lens") else 1
    acc = np.zeros((H, W, 4), np.float32)
    total = np.zeros((H, W, 4))
    for f in range(frames):
        pc = CC.push_constant(cam, H, case, f, 1)
        pc.flags |= abi.PT_USE_DLSS
        o.render_frame_dlss(fi, pc, acc)
        total += acc
    model = CC.make_model(cam, W, H, case, tris)
    off = CC.dlss_offset(fi)
    if not model.lens:
        fails = CC.check_dlss_point(model, acc, off, np.arange(H), name)
        assert not fails, "\n".join(fails)
        return
    ex = CC.Expectation(model, 1, frames, np.arange(H), max_mixed=LENS_PIXELS, dlss_offset=off)
    report = []
    fails = CC.check_image(ex, total / frames, name, report)
    print("\n".join(report))
    assert not fails, "\n".join(fails)
