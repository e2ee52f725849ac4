"""Cases shared by test_volume_expectation.py (the CPU oracle) and test_gpu_volume_expectation.py (the device): images of
synth_medium_box against the float64 expectation of tests/volref.py.

Pure absorbers with ior 1 return L T from every sample, so their pixels are checked one by one against the closed form,
within 1e-5 E.  Absorbers with ior 1.5 and scattering media are checked per channel over the face, as in estcases: the face
mean against E within 4.5 sigma + 1e-5 E, sigma from 64 interleaved batches of residuals.  Scattering media have no closed
form: E is volref's Monte Carlo, with its own standard error, and sigma is sqrt(sigma_img^2 + sigma_ref^2), required to be
<= 0.002 E.
"""
import functools
import math

import numpy as np

import estcases
import estref
import volref as V
from vk_gltf_renderer_b200 import synth

HALF = (4.0, 4.0, 0.5)     # the box: 8 x 8 wide, 1 deep
VIEW = 1.0                 # the camera sees [-1, 1]^2 of the +z face
BASE = dict(pbrBaseColorFactor=[1, 1, 1, 1], pbrMetallicFactor=0.0, pbrRoughnessFactor=0.0, transmissionFactor=1.0,
            thicknessFactor=1.0, specularFactor=1.0)
MS_GREY = 0.8              # multiscatter colour of the grey media: ssa(0.8) = 0.9906, so sigma_s ~ sigma_a


def grey_distance(tau, ms=MS_GREY, color=0.5):
    """attenuation distance for which the box depth (1) is `tau` extinction lengths"""
    return -math.log(color) * (1.0 + float(V.ssa(ms))) / tau


def material(color=(1, 1, 1), distance=None, ms=(0, 0, 0), g=0.0, ior=1.5, thickness=1.0):
    m = dict(BASE, ior=ior, thicknessFactor=thickness, attenuationColor=list(color), multiscatterColorFactor=list(ms),
             scatterAnisotropy=g)
    if distance is not None:
        m["attenuationDistance"] = distance
    return m


def medium(case):
    # a thin-walled material (thicknessFactor 0) still gets a medium: a transmission event toggles isInside and captures the
    # material's medium whatever its thickness (gltf_pathtrace.slang:396-403), so the segment between two thin walls is
    # attenuated; only the shadow ray's getShadowTransmission skips thin walls
    m = case["mat"]
    return V.Medium(m["attenuationColor"], m.get("attenuationDistance", float(np.finfo(np.float32).max)),
                    m["multiscatterColorFactor"], m["scatterAnisotropy"], rounded=case.get("rounded", True))


# ---- absorbers, ior 1: every sample is L T --------------------------------------------------------------------------------
ABSORB1 = {
    "grey": dict(mat=material((0.5,) * 3, 1.0, ior=1.0)),
    "chroma": dict(mat=material((0.9, 0.5, 0.05), 1.0, ior=1.0)),
    "channel0": dict(mat=material((0.6, 0.0, 0.3), 1.5, ior=1.0)),
    "distance0": dict(mat=material((0.999, 0.9995, 0.9999), 0.0, ior=1.0)),
    "distance_inf": dict(mat=material((0.5, 0.2, 0.1), math.inf, ior=1.0)),
    # absorbs (see medium()).  Unlike the ior-1 refraction (pdf +inf, a delta), the thin-walled lobe has a finite pdf, so the
    # environment-hit MIS weight pdf / (pdf + envW envPdf) drops below 1 on the rare samples whose half vector lies in the
    # GGX tail (tan > ~1e-3 at alpha 2e-6); surface NEE near the peak makes up for it in expectation.  So single samples are
    # not L T, and this case is checked by its face mean ("mean"), not pixel by pixel
    "thin_walled": dict(mat=material((0.5, 0.2, 0.1), 0.5, ior=1.0, thickness=0.0), mean=True),
    "tau8": dict(mat=material((math.exp(-8.0), math.exp(-4.0), math.exp(-1.0)), 1.0, ior=1.0)),
    "subnormal": dict(mat=material((0.99999, 0.999995, 0.99999), 1.0, ior=1.0)),
    "std_env_rot1.3": dict(mat=material((0.9, 0.5, 0.05), 1.0, ior=1.0), env="std_env", rotation=1.3),
}
# ---- absorbers, ior 1.5: internal reflections, cut by maxDepth ------------------------------------------------------------
ABSORB15 = {f"d{d}_spp{s}": dict(mat=material((0.7, 0.4, 0.2), 1.0), max_depth=d, spp=s) for d in (1, 2, 3, 5, 12) for s in (1, 4)}


# ---- scattering media ------------------------------------------------------------------------------------------------------
def _grey(g, tau, **kw):
    return dict(mat=material((0.5,) * 3, grey_distance(tau), (MS_GREY,) * 3, g), **kw)


def _threshold(k):
    # sigma_s = sigma_a ssa(ms) just below (k = 0) / above (k = 1) the walk's 0.001 threshold, sigma_a = ln 2 / 1
    target = 0.00097 if k == 0 else 0.00104
    ms = float(np.interp(target / math.log(2.0), V.ssa(np.linspace(0.0, 0.01, 10001)), np.linspace(0.0, 0.01, 10001)))
    return dict(mat=material((0.5,) * 3, 1.0, (ms,) * 3, 0.3))


SCATTER = {f"grey_g{g}_tau{t}": _grey(g, t) for g in (-0.5, 0.0, 0.3, 0.9) for t in (0.3, 3.0)}
SCATTER.update({
    # one channel nearly clear, the others ~50 extinction lengths: >= 64 scatters and the in-medium roulette.  A segment
    # that reaches the boundary is weighted exp((m - sigma_t) d), up to e^50 in the clear channel: its variance is
    # unbounded, so no mean converges: the case checks that the walk runs to the end without a device error, and reports
    "chroma_tau50": dict(mat=material((0.999, 0.01, 1e-4), 0.15, (0.9, 0.95, 0.99), 0.3), loose=True),
    "sigma_s_below": _threshold(0),
    "sigma_s_above": _threshold(1),
    # the environment's spread makes a sample noisier: 3 x the paths and frames
    "grey_std_env_rot1.3": _grey(0.3, 3.0, env="std_env", rotation=1.3, paths=3, frames=3),
    "grey_sphere_light": _grey(0.3, 3.0, intensity=0.0, lights="sphere"),
    "grey_point_light": _grey(0.3, 3.0, intensity=0.0, lights="point"),
})
MC_PATHS = 1_500_000


def lights(which):
    L = synth._light
    if which == "sphere":
        return [L("point", position=(0.5, 1.0, 6.0), color=(1.0, 0.9, 0.8), intensity=400.0, radius=2.0)]
    return [L("point", position=(0.5, 1.0, 6.0), color=(1.0, 0.9, 0.8), intensity=40.0)]


def scene(case):
    scn = synth.synth_medium_box(case["mat"], HALF, VIEW)
    scn.lights = lights(case["lights"]) if case.get("lights") else []
    return scn


def env_rgb(case):
    return estcases.std_env() if case.get("env") == "std_env" else estcases.furnace_env()


def lighting(case, env):
    return V.Lighting(env, case.get("rotation", 0.0), case.get("intensity", 1.0), lights(case["lights"]) if case.get("lights") else ())


def env_values(case, env):
    """environment radiance (times intensity) straight down and straight up"""
    lt = lighting(case, env)
    if not lt.env_on:
        return np.zeros(3), np.zeros(3)
    rgb, _ = lt.lookup(np.array([[0.0, 0.0, -1.0], [0.0, 0.0, 1.0]]))
    return rgb[0], rgb[1]


def absorber_E(case, env, rounded=True):
    down, up = env_values(case, env)
    med = medium(dict(case, rounded=rounded))
    ior = case["mat"]["ior"]
    return V.absorber_expectation(med, HALF[2], ior, case.get("max_depth", 5), down, up)


def environment(oracle_mod, case):
    """the estref.Env of the case's environment, with the alias table the CPU oracle builds"""
    o = oracle_mod.Oracle()
    o.set_environment(env_rgb(case))
    return estref.Env.from_oracle(o)


@functools.lru_cache(maxsize=None)
def scatter_E(oracle_mod, name):
    """volref's Monte Carlo for a SCATTER case, cached per session: (E [3], standard error [3])"""
    case = SCATTER[name]
    return V.monte_carlo(medium(case), lighting(case, environment(oracle_mod, case)), HALF, case["mat"]["ior"],
                         case.get("max_depth", 12), VIEW, MC_PATHS * case.get("paths", 1), seed=7)


def mask(ids):
    """the +z face (object id 1) eroded by the pixel filter's reach"""
    from scipy import ndimage
    st = np.ones((2 * estcases.FILTER_REACH + 1,) * 2, bool)
    return ndimage.binary_erosion(ids == 1, st, border_value=0)


def check_pixels(img, m, E, label, report, rtol=1e-5):
    """every pixel of the mask equals E within rtol E (absorbers with ior 1 behind refractions: every sample is E)"""
    vals = img[m][:, :3].astype(np.float64)
    E = np.asarray(E, np.float64)
    err = np.abs(vals - E).max(0)
    report.append(f"{label}: n={len(vals)} E={np.array2string(E, precision=7)} max|v-E|/E={np.array2string(err / np.maximum(E, 1e-300), precision=3)}")
    return bool(np.all(err <= rtol * E + 1e-30))


def check_mc(img, m, E, se_ref, label, report):
    """face mean against a Monte Carlo E: |mean - E| <= 4.5 sqrt(s_img^2 + s_ref^2) + 1e-5 E, and that sigma <= 0.002 E"""
    vals = img[m][:, :3].astype(np.float64)
    mean, s_img = estcases.batch_stats(vals)
    if not np.any(E):
        # nothing reaches the medium's NEE (a Dirac light alone): only the surfaces' NEE through their delta lobe, ~1e-9
        report.append(f"{label}: n={len(vals)} mean={np.array2string(mean, precision=3)} E=0")
        return bool(np.all(np.abs(mean) < 1e-5)), True
    s = np.sqrt(s_img ** 2 + np.asarray(se_ref) ** 2)
    dev = np.abs(mean - E) / np.maximum(s, 1e-300)
    report.append(f"{label}: n={len(vals)} mean={np.array2string(mean, precision=5)} E={np.array2string(E, precision=5)} "
                  f"sigma/E={np.array2string(s / np.maximum(E, 1e-300), precision=5)} |d|/sigma={np.array2string(dev, precision=2)}")
    return bool(np.all(np.abs(mean - E) <= estcases.N_SIGMA * s + 1e-5 * E)), bool(np.all(s <= estcases.MAX_REL_SIGMA * E))
