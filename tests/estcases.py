"""Cases and statistics shared by test_estimator_expectation.py (the CPU oracle) and test_gpu_estimator_expectation.py (the
device): rendered images of synth_furnace_polyhedron / synth_enclosure against the float64 expectation of tests/estref.py.

A case renders `frames` frames into the running mean.  The seed of a sample is xxhash32(x, y, frame), so the pixels of a face
are independent draws of the same estimator; their residuals value - E (E per face, or per pixel where a light is at a
finite distance) are dealt, in raster order, into B interleaved batches.  Per face and channel the test takes the batch means,
their standard error sigma, and asserts |mean - E| <= 4.5 sigma + 1e-5 E, and that sigma <= 0.002 E, so that a bias of 1 %
would stand at >= 5 sigma.  Faces are masked by the frame-0 object ids, eroded by the reach of the pixel filter.
"""
import math
import os

import numpy as np
from scipy import ndimage

import bsdfref as R
import estref
from vk_gltf_renderer_b200 import camera as camm
from vk_gltf_renderer_b200 import synth

ASSETS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "assets")
BATCHES = 64
N_SIGMA = 4.5
MAX_REL_SIGMA = 0.002     # 1 % / 5 sigma
# The clamp threshold: far above any sample (asserted per case from the running mean), so the clamp never fires.
NO_CLAMP = 3.0e38
# Gaussian pixel filter (b200pt.cu:206-209, pt_oracle.cpp:2169-2173): sigma 0.4246609 px, radius sqrt(-2 ln max(1e-38, u)) is
# at most sqrt(-2 ln 1e-38) = 13.24 sigma, so a sample lands within 0.5 + 5.62 px of its pixel's corner: 7 px covers it.
FILTER_REACH = math.ceil(0.5 + math.sqrt(-2.0 * math.log(1e-38)) * 0.4246609)

LAMBERT = lambda rho: dict(pbrBaseColorFactor=[rho, rho, rho, 1.0], pbrMetallicFactor=0.0, pbrRoughnessFactor=1.0, specularFactor=0.0)
METAL = lambda alpha: dict(pbrBaseColorFactor=[1.0, 1.0, 1.0, 1.0], pbrMetallicFactor=1.0, pbrRoughnessFactor=math.sqrt(alpha))
FURNACE_L = (0.9, 0.6, 0.3)


def furnace_env():
    return np.broadcast_to(np.asarray(FURNACE_L, np.float32), (32, 64, 3)).copy()


def spot_env():
    """256 x 128, dim (0.02, 0.03, 0.04), one 3 x 2-texel block 1e4 x brighter, one isolated texel 300 x brighter"""
    e = np.empty((128, 256, 3), np.float32)
    e[:] = (0.02, 0.03, 0.04)
    e[20:22, 40:43] = np.float32(1e4) * e[40, 100]
    e[90, 30] = (6.0, 4.5, 3.0)
    return e


def std_env():
    from vk_gltf_renderer_b200 import hdr
    return hdr.load_hdr(os.path.join(ASSETS, "std_env.hdr"))


def lights(which):
    L = synth._light
    allfive = {
        "point": L("point", position=(2.0, 2.5, 4.0), color=(1.0, 0.9, 0.8), intensity=30.0),
        "sphere": L("point", position=(-1.5, 2.0, 3.5), color=(0.6, 0.8, 1.0), intensity=25.0, radius=0.6),
        "spot": L("spot", position=(0.5, 3.0, 4.0), direction=(-0.1, -0.6, -0.8), color=(1, 1, 1), intensity=60.0, rng=9.0,
                  inner=0.3, outer=0.9),
        "directional": L("directional", direction=(-0.3, -0.5, -1.0), color=(1.0, 0.95, 0.9), intensity=1.5),
        "directional_cone": L("directional", direction=(0.4, -0.6, -0.9), color=(0.4, 0.5, 0.7), intensity=2.0, angular_size=0.25),
    }
    return list(allfive.values()) if which == "all" else [allfive[which]]


# name -> dict(mat: add_material keywords, env, rotation, intensity, lights, frames: the oracle's frame count)
FURNACE = {f"furnace_lambert_{r}": dict(mat=LAMBERT(r), env="furnace", frames=80) for r in (0.3, 1.0)}
FURNACE.update({f"furnace_ggx_{a}": dict(mat=METAL(a), env="furnace", frames=250) for a in (0.05, 0.3, 0.8)})
ENVLIT = {f"{e}_{m}_rot{rot}": dict(mat=LAMBERT(0.8) if m == "lambert" else METAL(0.3), env=e, rotation=rot, frames=f)
          for e, f in (("std_env", 400), ("spot_env", 1200)) for m in ("lambert", "ggx0.3") for rot in (0.0, 1.3)}
LIGHTS = {f"light_{w}": dict(mat=LAMBERT(0.8), env="furnace", intensity=0.0, lights=w, frames=160)
          for w in ("point", "sphere", "spot", "directional", "directional_cone", "all")}
# all five lights under the constant environment: light and environment techniques at 0.5 / 0.5
LIGHTS["light_all_env"] = dict(mat=LAMBERT(0.8), env="furnace", lights="all", frames=480)
POLY_CASES = {**FURNACE, **ENVLIT, **LIGHTS}
ENCLOSURE_CASES = [(rho, d, s) for rho in (0.5, 0.9) for d in (2, 4, 12) for s in (1, 4)]
ENCLOSURE_E = (0.7, 0.5, 0.3)

_ENVS = {"furnace": furnace_env, "spot_env": spot_env, "std_env": std_env}


def env_rgb(case):
    return _ENVS[case["env"]]()


def poly_scene(case):
    scn, normals = synth.synth_furnace_polyhedron([case["mat"]])
    scn.lights = lights(case["lights"]) if case.get("lights") else []
    return scn, normals


def frame_info(scn, w, h, case):
    return camm.make_frame_info(scn.camera, w, h, env_rotation=case.get("rotation", 0.0), env_intensity=case.get("intensity", 1.0))


# ---- geometry of the orthographic view -------------------------------------------------------------------------------------
def view_dir(cam):
    """unit direction from the scene towards the camera"""
    d = np.asarray(cam.eye, np.float64) - np.asarray(cam.center, np.float64)
    return d / np.linalg.norm(d)


def pixel_points(cam, w, h, normal, point, ys, xs):
    """world position, on the plane (normal, point), of the ray through the centre of each pixel (ys, xs)"""
    view = camm.look_at(cam.eye, cam.center, cam.up)
    proj = camm.ortho_vk(cam.xmag, cam.ymag, cam.znear, cam.zfar)
    clip = np.stack([(xs + 0.5) / w * 2 - 1, (ys + 0.5) / h * 2 - 1, -np.ones(len(xs)), np.ones(len(xs))], -1)
    vc = clip @ np.linalg.inv(proj).T
    o = (vc / vc[:, 3:]) @ np.linalg.inv(view).T
    o = o[:, :3]
    d = -view_dir(cam)
    t = ((np.asarray(point) - o) @ normal) / (d @ normal)
    return o + t[:, None] * d


def face_masks(ids, min_pixels):
    """{face k: eroded mask} for the faces whose eroded mask keeps at least `min_pixels` pixels"""
    st = np.ones((2 * FILTER_REACH + 1,) * 2, bool)
    out = {}
    for k in range(20):
        m = ndimage.binary_erosion(ids == k + 1, st, border_value=0)
        if m.sum() >= min_pixels:
            out[k] = m
    return out


def batch_stats(values, batches=BATCHES):
    """values [n, 3] in raster order -> (mean [3] of all values, sigma [3] from the spread of `batches` interleaved batch
    means)"""
    means = np.stack([values[b::batches].mean(0) for b in range(batches)])
    return values.mean(0), means.std(0, ddof=1) / math.sqrt(batches)


def expected_face(case, env, scn, normals, k, mask, w, h, sub=4):
    """E of face k: the shading-point expectation, one rgb per face, or with lights at a finite distance one per pixel of
    the mask (raster order) at the pixel's centre"""
    n = normals[k]
    v = view_dir(scn.camera)
    mat = case["mat"]
    lobe = R.METAL if mat["pbrMetallicFactor"] == 1.0 else R.DIFFUSE
    alpha = mat["pbrRoughnessFactor"] ** 2
    b = estref.Bsdf(n, v, lobe, base=mat["pbrBaseColorFactor"][:3], alpha=alpha)
    intensity = case.get("intensity", 1.0)
    if case["env"] == "furnace" and intensity > 0 and not case.get("lights"):
        return np.asarray(FURNACE_L) * b.albedo()
    if not case.get("lights"):
        # std_env's 1500 x 750 texels are 0.24 degrees wide: 2 x 2 nodes resolve their bilinear patches (halving checked)
        sub = 2 if env.w > 1000 else sub
        return estref.expectation(b, env=env, env_rotation=case.get("rotation", 0.0), env_intensity=intensity, sub=sub)
    ys, xs = np.nonzero(mask)
    verts, faces = synth.icosahedron()
    pts = pixel_points(scn.camera, w, h, n, verts[faces[k][0]], ys, xs)
    kw = dict(env=env if intensity > 0 else None, env_intensity=intensity, lights=scn.lights, cone_n=(32, 32))
    e_env = estref.expectation(b, pos=pts[0], parts=True, **kw)
    e_lights = [estref.expectation(b, pos=p, env_terms=False, **kw) for p in pts]
    return e_env["env_nee"] + e_env["bsdf_env"] + np.asarray(e_lights)


def check_face(img, mask, E, label, report):
    """E: rgb [3] or per pixel [n, 3].  sigma comes from the residuals value - E, so a face whose expectation varies across
    it is not taken for noise; the reported E is the mean over the face"""
    vals = img[mask][:, :3].astype(np.float64)
    E_pix = np.broadcast_to(np.asarray(E, np.float64), vals.shape)
    E = E_pix.mean(0)
    resid, sigma = batch_stats(vals - E_pix)
    mean = E + resid
    dev = np.abs(mean - E) / np.maximum(sigma, 1e-300)
    rel = sigma / np.maximum(np.abs(E), 1e-300)
    report.append(f"{label}: n={len(vals)} mean={np.array2string(mean, precision=5)} E={np.array2string(E, precision=5)} "
                  f"sigma/E={np.array2string(rel, precision=5)} |d|/sigma={np.array2string(dev, precision=2)}")
    ok_val = np.all(np.abs(mean - E) <= N_SIGMA * sigma + 1e-5 * E)
    ok_sens = np.all(sigma <= MAX_REL_SIGMA * E)
    return ok_val, ok_sens


def assert_no_clamp(img, frames, spp):
    """the accumulated image is the mean of frames * spp non-negative samples, so none exceeded frames * spp * max(mean)"""
    lum = img[..., :3].astype(np.float64).mean(-1)
    assert np.isfinite(img).all()
    assert frames * spp * lum.max() < NO_CLAMP
