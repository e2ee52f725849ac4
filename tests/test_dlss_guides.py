"""The DLSS variant without a GPU: the host mirror's Halton jitter, the DEVICE arithmetic (csrc/dlss_guides.cuh) compiled for the
host against the oracle's independent restatement and float64, and known answers of the oracle's six guide images on a synthetic
scene (a camera-facing diffuse quad, a mirror facing a diffuse wall, open sky).  The oracle's DLSS variant is tests/dlss_oracle.cpp."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest

from dlss_oracle import DlssOracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
CSRC = os.path.join(ROOT, "vk_gltf_renderer_b200", "csrc")
CUDA_INC = os.environ.get("CUDA_HOME", "/usr/local/cuda") + "/include"
W = H = 32


# ---- Halton jitter ------------------------------------------------------------------------------------------------------------
def halton64(index):
    """shaderio::halton in float64: one loop over both bases that stops when either remainder reaches 0"""
    sx = sy = float(index)
    ax, ay, az, aw = 1.0, 1.0, 0.0, 0.0
    while sx > 0 and sy > 0:
        ax /= 2.0
        ay /= 3.0
        az += ax * math.fmod(sx, 2.0)
        aw += ay * math.fmod(sy, 3.0)
        sx, sy = math.floor(sx / 2.0), math.floor(sy / 3.0)
    return az, aw


def test_dlss_jitter_follows_halton():
    from vk_gltf_renderer_b200 import camera as camm
    f, third = np.float32, np.float32(1.0) / np.float32(3.0)
    assert camm.dlss_jitter(1) == (0.0, third - f(0.5))                       # (0, -1/6)
    assert camm.dlss_jitter(2) == (-0.5, third * f(2.0) - f(0.5))             # base 2 stops after one digit: x = 0
    assert camm.dlss_jitter(3) == (0.25, third / f(3.0) - f(0.5))
    for i in range(1, 65):
        jx, jy = camm.dlss_jitter(i)
        hx, hy = halton64(i)
        assert abs(jx - (hx - 0.5)) <= 1e-6 and abs(jy - (hy - 0.5)) <= 1e-6, i
        assert -0.5 <= jx < 0.5 and -0.5 <= jy < 0.5


# ---- device arithmetic on the host ---------------------------------------------------------------------------------------------
def env_brdf64(spec, alpha, nov):
    nov = abs(nov)
    X = np.array([1.0, nov, nov * nov, nov ** 3])
    Y = np.array([1.0, alpha, alpha * alpha, alpha ** 3])
    M1 = np.array([[0.99044, -1.28514], [1.29678, -0.755907]])
    M2 = np.array([[1.0, 2.92338, 59.4188], [20.3225, -27.0302, 222.592], [121.563, 626.13, 316.627]])
    M3 = np.array([[0.0365463, 3.32707], [9.0632, -9.04756]])
    M4 = np.array([[1.0, 3.59685, -1.36772], [9.04401, -16.3174, 9.22949], [5.56589, 19.7886, -20.2123]])
    bias = (M1 @ X[[0, 1]]) @ Y[[0, 1]] / ((M2 @ X[[0, 1, 3]]) @ Y[[0, 1, 3]])
    scale = (M3 @ X[[0, 1]]) @ Y[[0, 1]] / ((M4 @ X[[0, 2, 3]]) @ Y[[0, 1, 3]])
    bias *= min(max(spec[1] * 50.0, 0.0), 1.0)
    return np.asarray(spec, np.float64) * max(0.0, scale) + max(0.0, bias)


def motion64(curr, prev, prev_mvp, curr_mvp, res):
    c = np.asarray(curr, np.float64) @ np.asarray(curr_mvp, np.float64).reshape(4, 4)
    p = np.asarray(prev, np.float64) @ np.asarray(prev_mvp, np.float64).reshape(4, 4)
    return (p[:2] / p[3] - c[:2] / c[3]) * 0.5 * np.asarray(res, np.float64)


@pytest.fixture(scope="module")
def host_dlss(tmp_path_factory):
    if not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")):
        pytest.skip("CUDA headers not found")
    exe = str(tmp_path_factory.mktemp("dlss") / "host_dlss_check")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-I" + CUDA_INC, "-o", exe, os.path.join(CSRC, "tools", "host_dlss_check.cpp")])

    def run(mode, data, out_dtype):
        d = os.path.dirname(exe)
        np.ascontiguousarray(data, np.float32).tofile(os.path.join(d, "in.bin"))
        subprocess.check_call([exe, mode, os.path.join(d, "in.bin"), os.path.join(d, "out.bin")])
        return np.fromfile(os.path.join(d, "out.bin"), out_dtype)
    return run


def test_env_brdf_approx2_device_source_matches_oracle_and_float64(host_dlss, oracle_mod):
    rng = np.random.default_rng(7)
    n = 4000
    rec = np.concatenate([rng.random((n, 3)) * rng.choice([0.02, 0.2, 1.0], (n, 1)), rng.random((n, 1)),
                          rng.uniform(-1, 1, (n, 1))], 1).astype(np.float32)
    rec[:8, 3] = [0, 1, 0, 1, 0.5, 0.5, 1e-4, 0.999]   # alpha at the ends, NoV at the ends
    rec[:8, 4] = [0, 0, 1, 1, -1, 1e-3, 0.5, -0.2]
    rec[8:12, :3] = 0.0                                  # specular reflectance 0: the bias hack
    dev = host_dlss("brdf", rec, np.float32).reshape(n, 3)
    ref = DlssOracle().env_brdf_approx2(rec)
    assert np.array_equal(dev.view(np.uint32), ref.view(np.uint32))
    exp = np.array([env_brdf64(r[:3], r[3], r[4]) for r in rec.astype(np.float64)])
    assert np.all(np.abs(ref - exp) <= 1e-5 * np.maximum(np.abs(exp), 1e-2))


def test_motion_vector_device_source_matches_oracle_and_float64(host_dlss, oracle_mod):
    from vk_gltf_renderer_b200 import camera as camm
    from vk_gltf_renderer_b200.scene import Camera
    rng = np.random.default_rng(8)
    cam = Camera()
    cam.eye, cam.center, cam.yfov, cam.znear, cam.zfar = np.array([0.3, 1.0, 5.0], np.float32), np.zeros(3, np.float32), math.radians(50), 0.1, 100.0
    curr = np.array(camm.make_frame_info(cam, 64, 48).viewProjMatrix, np.float32)
    cam.eye = np.array([0.45, 0.9, 4.7], np.float32)
    cam.center = np.array([0.05, 0.02, 0.0], np.float32)
    prev = np.array(camm.make_frame_info(cam, 64, 48).viewProjMatrix, np.float32)
    n = 3000
    pts = rng.uniform(-2, 2, (n, 3))
    w = (rng.random(n) < 0.8).astype(np.float64)      # surfaces (w = 1) and sky directions (w = 0)
    pts[w == 0] = pts[w == 0] / np.linalg.norm(pts[w == 0], axis=1, keepdims=True) * np.array([1, 1, 0]) + np.array([0, 0, -1.5])
    moved = pts + rng.normal(0, 0.05, (n, 3)) * w[:, None]
    rec = np.concatenate([pts, w[:, None], moved, w[:, None], np.tile([64.0, 48.0], (n, 1))], 1).astype(np.float32)
    dev = host_dlss("motion", np.concatenate([prev, curr, rec.reshape(-1)]), np.float32).reshape(n, 2)
    ref = DlssOracle().motion_vector(rec, prev, curr)
    assert np.array_equal(dev.view(np.uint32), ref.view(np.uint32))
    for r, got in zip(rec.astype(np.float64), ref.astype(np.float64)):
        exp = motion64(r[0:4], r[4:8], prev.astype(np.float64), curr.astype(np.float64), r[8:10])
        c = r[0:4] @ curr.astype(np.float64).reshape(4, 4)
        scale = (np.abs(c[:2] / c[3]) + 1.0) * r[8:10]   # the NDC terms whose difference the motion is
        assert np.all(np.abs(got - exp) <= 1e-5 * scale), (r, got, exp)


def test_binary16_and_unorm8_rounding(host_dlss):
    x = np.concatenate([np.float32([0, 1, -1, 0.5, 65504, 65519.99, 65520, 1e-8, 6e-5, 2.0 ** -25, 3 * 2.0 ** -26, 127.5 / 255, 0.2 / 255]),
                        np.random.default_rng(9).uniform(-2, 2, 5000).astype(np.float32)]).astype(np.float32)
    out = host_dlss("pack", x, np.uint8)
    halfs = out[:2 * len(x)].view(np.uint16)
    unorm = out[2 * len(x):].view(np.uint32)
    with np.errstate(over="ignore"):
        assert np.array_equal(halfs, x.astype(np.float16).view(np.uint16))   # numpy: round to nearest even
    exp = np.floor(np.clip(x, 0, 1).astype(np.float32) * np.float32(255) + 0.5)
    assert np.array_equal(unorm, exp.astype(np.uint32))


# ---- oracle known answers -------------------------------------------------------------------------------------------------------
def _quad(scn, x0, x1, y0, y1, z, normal_z, mat, matrix=None):
    pos = [[x0, y0, z], [x1, y0, z], [x1, y1, z], [x0, y1, z]]
    idx = [[0, 1, 2], [0, 2, 3]] if normal_z > 0 else [[0, 2, 1], [0, 3, 2]]
    prim = scn.add_primitive(pos, idx, normals=[[0, 0, normal_z]] * 4, uv0=[[0, 0], [1, 0], [1, 1], [0, 1]])
    return scn.add_node(prim, mat, matrix=matrix)


def kat_scene(quad_offset=(0.0, 0.0, 0.0)):
    """camera at z = 5 looking down -z; a diffuse quad (node 0) at z = 0 left of centre, a mirror (node 1) at z = 0 right of
    centre facing the camera, and a diffuse wall (node 2) behind the camera at z = 8 facing -z that catches the mirror's
    reflections with x < 2.6; everything else is open sky"""
    from vk_gltf_renderer_b200.scene import Camera, Scene
    scn = Scene()
    # specularFactor 0: no dielectric specular lobe, so the quad's samples are diffuse reflections only
    diffuse = scn.add_material(pbrBaseColorFactor=[0.6, 0.4, 0.2, 1], pbrRoughnessFactor=1.0, pbrMetallicFactor=0.0, specularFactor=0.0)
    mirror = scn.add_material(pbrBaseColorFactor=[1, 1, 1, 1], pbrRoughnessFactor=0.0, pbrMetallicFactor=1.0)
    wall = scn.add_material(pbrBaseColorFactor=[0.5, 0.5, 0.5, 1], pbrRoughnessFactor=1.0, pbrMetallicFactor=0.0)
    m = np.eye(4)
    m[:3, 3] = quad_offset
    _quad(scn, -1.5, -0.5, -0.5, 0.5, 0.0, 1, diffuse, m)
    _quad(scn, 0.5, 1.5, -0.5, 0.5, 0.0, 1, mirror)
    _quad(scn, 0.0, 2.6, -4.0, 4.0, 8.0, -1, wall)
    cam = Camera()
    cam.eye, cam.center = np.array([0, 0, 5], np.float32), np.zeros(3, np.float32)
    cam.yfov, cam.znear, cam.zfar = math.radians(45.0), 0.1, 100.0
    scn.camera = cam
    return scn


def const_env():
    return np.full((16, 32, 3), 0.5, np.float32)


def dlss_frame(cam, index, frame_count0=0, prev_vp=None):
    from vk_gltf_renderer_b200 import abi, camera as camm
    fi = camm.make_frame_info(cam, W, H)
    if prev_vp is not None:
        fi.prevMVP[:] = list(prev_vp)
    fi.jitter[:] = list(camm.dlss_jitter(index))
    pc = camm.make_push_constant(cam, H, frame_count=frame_count0, total_samples=0, num_samples=1, max_depth=4)
    pc.frameCount = index
    pc.flags |= abi.PT_USE_DLSS
    return fi, pc


def primary_hits(fi):
    """float64 primary rays through the jittered pixel positions, intersected with z = 0: (points [H, W, 3], directions)"""
    pinv = np.asarray(fi.projInv, np.float64).reshape(4, 4)
    vinv = np.asarray(fi.viewInv, np.float64).reshape(4, 4)
    ys, xs = np.mgrid[0:H, 0:W].astype(np.float64)
    cx = (xs + 0.5 + fi.jitter[0]) / W * 2 - 1
    cy = (ys + 0.5 + fi.jitter[1]) / H * 2 - 1
    v = np.stack([cx, cy, -np.ones_like(cx), np.ones_like(cx)], -1) @ pinv
    v = v / v[..., 3:]
    org = vinv[3, :3]
    d = (v @ vinv)[..., :3] - org
    d /= np.linalg.norm(d, axis=-1, keepdims=True)
    t = -org[2] / d[..., 2]
    return org + d * t[..., None], d


def project(p, vp):
    c = np.concatenate([p, np.ones(p.shape[:-1] + (1,))], -1) @ np.asarray(vp, np.float64).reshape(4, 4)
    return c[..., :2] / c[..., 3:]


@pytest.fixture(scope="module")
def kat(oracle_mod):
    o = DlssOracle()
    scn = kat_scene()
    o.set_scene(scn)
    o.set_environment(const_env())
    return o, scn


def regions(pts):
    quad = (pts[..., 0] > -1.49) & (pts[..., 0] < -0.51) & (np.abs(pts[..., 1]) < 0.49)
    mirror = (pts[..., 0] > 0.51) & (pts[..., 0] < 1.49) & (np.abs(pts[..., 1]) < 0.49)
    return quad, mirror


def test_static_camera_has_zero_motion(kat):
    o, scn = kat
    accum = np.zeros((H, W, 4), np.float32)
    fi, pc = dlss_frame(scn.camera, 1)
    g1 = o.render_frame_dlss(fi, pc, accum)
    fi2, pc2 = dlss_frame(scn.camera, 2, 1, prev_vp=fi.viewProjMatrix)
    g2 = o.render_frame_dlss(fi2, pc2, accum)
    for g in (g1, g2):
        assert np.all(g["motion"] == 0)
    pts, _ = primary_hits(fi2)
    quad, mirror = regions(pts)
    assert quad.sum() > 50 and mirror.sum() > 50
    sky = g2["depth"] == 1.0
    assert sky.sum() > 100 and np.all(g2["albedo"][sky] == 0) and np.all(g2["normal_roughness"][sky] == 0)
    assert np.all(g2["albedo"][quad] == [153, 102, 51, 255])       # binary16 of (0.6, 0.4, 0.2) -> UNORM8, solid
    assert np.all(g2["normal_roughness"][quad] == np.float16([0, 0, 1, 1]))
    assert np.all(g2["spec_albedo"][sky] == np.float16([0, 0, 0, 1]))


def test_camera_translation_moves_surfaces_not_the_sky(kat):
    o, scn = kat
    from vk_gltf_renderer_b200 import camera as camm
    accum = np.zeros((H, W, 4), np.float32)
    fi1, pc1 = dlss_frame(scn.camera, 1)
    o.render_frame_dlss(fi1, pc1, accum)
    cam2 = kat_scene().camera
    cam2.eye = cam2.eye + np.float32([0.1, 0.05, 0])
    cam2.center = cam2.center + np.float32([0.1, 0.05, 0])
    fi2, pc2 = dlss_frame(cam2, 2, 1, prev_vp=fi1.viewProjMatrix)
    g = o.render_frame_dlss(fi2, pc2, accum)
    sky = g["depth"] == 1.0
    assert sky.sum() > 100 and np.all(g["motion"][sky] == 0)
    pts, _ = primary_hits(fi2)
    quad, _ = regions(pts)
    exp = (project(pts, fi1.viewProjMatrix) - project(pts, fi2.viewProjMatrix)) * 0.5 * np.array([W, H])
    got = g["motion"].astype(np.float64)
    assert np.abs(exp[quad]).max() > 0.3
    assert np.all(np.abs(got[quad] - exp[quad]) <= 1e-2)
    assert camm.make_frame_info(cam2, W, H).viewProjMatrix[:] == fi2.viewProjMatrix[:]


def test_instance_motion_follows_the_previous_transforms(oracle_mod):
    o = DlssOracle()
    before = kat_scene()
    o.set_environment(const_env())
    prev = np.stack([np.asarray(rn["objectToWorld"], np.float32) for rn in before.render_nodes])
    moved = kat_scene(quad_offset=(0.12, -0.07, 0.0))
    o.set_scene(moved)
    cam = moved.camera
    accum = np.zeros((H, W, 4), np.float32)
    fi, pc = dlss_frame(cam, 3)
    g = o.render_frame_dlss(fi, pc, accum, prev_object_to_world=prev)
    pts, _ = primary_hits(fi)
    quad = (pts[..., 0] > -1.37) & (pts[..., 0] < -0.39) & (np.abs(pts[..., 1] + 0.07) < 0.49)
    _, mirror = regions(pts)
    exp = (project(pts - np.array([0.12, -0.07, 0.0]), fi.viewProjMatrix) - project(pts, fi.viewProjMatrix)) * 0.5 * np.array([W, H])
    got = g["motion"].astype(np.float64)
    assert quad.sum() > 50 and np.abs(exp[quad]).max() > 0.3
    assert np.all(np.abs(got[quad] - exp[quad]) <= 1e-2)
    assert np.all(got[mirror] == 0) and np.all(got[g["depth"] == 1.0] == 0)
    # the next frame has no update before it: no previous transforms, camera-only (here: no) motion
    fi2, pc2 = dlss_frame(cam, 4, 1, prev_vp=fi.viewProjMatrix)
    assert np.all(o.render_frame_dlss(fi2, pc2, accum)["motion"] == 0)


def test_specular_hit_distance_and_albedo(kat):
    o, scn = kat
    accum = np.zeros((H, W, 4), np.float32)
    fi, pc = dlss_frame(scn.camera, 5)
    g = o.render_frame_dlss(fi, pc, accum)
    pts, d = primary_hits(fi)
    quad, mirror = regions(pts)
    # mirror: the reflected ray (d.x, d.y, -d.z) from z = 0 reaches the wall z = 8 at t = 8 / -d.z unless x leaves [0, 2.6]
    t = 8.0 / -d[..., 2]
    xw = pts[..., 0] + d[..., 0] * t
    to_wall = mirror & (xw < 2.58) & (np.abs(pts[..., 1] + d[..., 1] * t) < 3.9)
    to_sky = mirror & (xw > 2.62)
    assert to_wall.sum() > 20 and to_sky.sum() > 20
    dist = g["spec_hit_dist"].astype(np.float64)
    exp16 = t.astype(np.float16).astype(np.float64)
    ulp = np.spacing(exp16.astype(np.float16)).astype(np.float64)
    assert np.all(np.abs(dist[to_wall] - exp16[to_wall]) <= ulp[to_wall])    # the ray leaves a safeOffsetRay point
    assert np.mean(dist[to_wall] == exp16[to_wall]) > 0.9
    assert np.all(dist[to_sky] == 65504.0)
    assert np.all(dist[quad] == 0) and np.all(dist[g["depth"] == 1.0] == 0)
    # specular albedo of both materials: dielectric f0 (ior 1.5) x specular colour 1, at the guide's roughness and N = +z
    for region in (quad, mirror):
        nr = g["normal_roughness"][region].astype(np.float64)
        assert np.all(nr[:, :3] == [0, 0, 1])
        for (alpha, nov), got in zip(zip(nr[:, 3], d[region][:, 2]), g["spec_albedo"][region].astype(np.float64)):
            exp = env_brdf64(np.full(3, 0.04), alpha, nov)
            assert np.all(np.abs(got[:3] - exp) <= 2e-3 * exp + 1e-7) and got[3] == 1.0


def test_dlss_frames_replace_the_image(kat):
    o, scn = kat
    a = np.zeros((H, W, 4), np.float32)
    fi1, pc1 = dlss_frame(scn.camera, 1)
    o.render_frame_dlss(fi1, pc1, a)
    fi2, pc2 = dlss_frame(scn.camera, 2, 1, prev_vp=fi1.viewProjMatrix)
    g = o.render_frame_dlss(fi2, pc2, a)
    b = np.full((H, W, 4), 7.0, np.float32)
    g_alone = o.render_frame_dlss(fi2, pc2, b)
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    for k in g:
        assert np.array_equal(g[k], g_alone[k]), k
    assert np.all(a[..., 3][g["depth"] == 1.0] == 0) and np.all(a[..., 3][g["depth"] < 1.0] > 0)


def test_dlss_frame_refusals(kat):
    from vk_gltf_renderer_b200 import abi
    o, scn = kat
    accum = np.zeros((H, W, 4), np.float32)
    fi, pc = dlss_frame(scn.camera, 1)
    pc.numSamples = 2
    with pytest.raises(ValueError):
        o.render_frame_dlss(fi, pc, accum)
    pc.numSamples = 1
    pc.flags &= ~abi.PT_USE_DLSS
    with pytest.raises(ValueError):
        o.render_frame_dlss(fi, pc, accum)   # a plain frame is not the DLSS variant
