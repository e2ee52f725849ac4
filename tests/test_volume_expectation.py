"""The CPU oracle's images of a medium box converge to the float64 expectation of the participating-media estimator
(tests/volref.py): absorbers with ior 1 pixel by pixel, absorbers with ior 1.5 over maxDepth and ptSamples, and scattering
media against volref's Monte Carlo.  See tests/volcases.py.  The device runs the same cases in
test_gpu_volume_expectation.py."""
import numpy as np
import pytest

import estcases
import volcases as VC
from vk_gltf_renderer_b200 import camera as camm

W = H = 96
# the scattering cases the oracle runs (the device runs all of them): both optical depths, backward and forward phase,
# a Dirac light and the threshold of the walk
ORACLE_SCATTER = ["grey_g-0.5_tau3.0", "grey_g0.9_tau0.3", "grey_point_light", "sigma_s_above"]


def _render(O, case, frames, max_depth=5, spp=1):
    scn = VC.scene(case)
    o = O.Oracle()
    o.set_scene(scn)
    o.set_environment(VC.env_rgb(case))
    fi = camm.make_frame_info(scn.camera, W, H, env_rotation=case.get("rotation", 0.0), env_intensity=case.get("intensity", 1.0))
    acc = np.zeros((H, W, 4), np.float32)
    ids = np.zeros((H, W), np.uint32)
    for f in range(frames):
        pc = camm.make_push_constant(scn.camera, H, frame_count=f, total_samples=f * spp, num_samples=spp, max_depth=max_depth,
                                     firefly_clamp=estcases.NO_CLAMP)
        o.render_frame(fi, pc, acc, object_id=ids if f == 0 else None)
    estcases.assert_no_clamp(acc, frames, spp)
    return acc, VC.mask(ids)


@pytest.mark.parametrize("name", sorted(VC.ABSORB1))
def test_absorber_ior1(oracle_mod, name):
    case = VC.ABSORB1[name]
    acc, m = _render(oracle_mod, case, 2)
    env = VC.environment(oracle_mod, case)
    E = VC.absorber_E(case, env)
    report = []
    if case.get("mean"):
        ok, ok_sens = estcases.check_face(acc, m, E, f"absorber {name} (face mean)", report)
        ok = ok and ok_sens
    else:
        ok = VC.check_pixels(acc, m, E, f"absorber {name}", report)
    print(report[0])
    assert m.sum() > 4000
    assert ok, report[0]


def test_absorber_half_rounding_is_pinned(oracle_mod):
    """at least one case tells the binary16 coefficients from full-precision ones by >= 50 x the tolerance"""
    env = VC.environment(oracle_mod, VC.ABSORB1["grey"])
    gaps = {}
    for name, case in VC.ABSORB1.items():
        if case.get("env"):
            continue
        E, Eu = VC.absorber_E(case, env), VC.absorber_E(case, env, rounded=False)
        gaps[name] = float(np.max(np.abs(E - Eu) / np.maximum(E, 1e-300)))
    print(gaps)
    assert max(gaps.values()) >= 50 * 1e-5


@pytest.mark.parametrize("name", sorted(VC.ABSORB15))
def test_absorber_ior15(oracle_mod, name):
    case = VC.ABSORB15[name]
    spp = case["spp"]
    # maxDepth 2 returns F L with probability F = 0.04: 20 x the samples for sigma <= 0.002 E
    acc, m = _render(oracle_mod, case, (1600 if case["max_depth"] == 2 else 48) // spp, max_depth=case["max_depth"], spp=spp)
    E = VC.absorber_E(case, VC.environment(oracle_mod, case))
    report = []
    if not E.any():
        # maxDepth 1: the first hit is the only bounce; its surface NEE through a delta lobe adds ~1e-9 (oracle) to ~1e-6 (device)
        assert np.abs(acc[m][:, :3]).mean() < 1e-5
        return
    ok_val, ok_sens = estcases.check_face(acc, m, E, f"absorber ior 1.5 {name}", report)
    print(report[0])
    assert ok_val, report[0]
    assert ok_sens, report[0]


@pytest.mark.parametrize("name", ORACLE_SCATTER)
def test_scattering(oracle_mod, name):
    case = VC.SCATTER[name]
    acc, m = _render(oracle_mod, case, 240, max_depth=case.get("max_depth", 12))
    E, se = VC.scatter_E(oracle_mod, name)
    report = []
    ok_val, ok_sens = VC.check_mc(acc, m, E, se, f"scattering {name}", report)
    print(report[0])
    assert ok_val, report[0]
    assert ok_sens, report[0]
