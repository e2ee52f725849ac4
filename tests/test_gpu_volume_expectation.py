"""The device's images of a medium box converge to the float64 expectation of the participating-media estimator
(tests/volref.py): the cases of test_volume_expectation.py at a larger image and every scattering case, rendered through
render_headless, plus frame batch 3 and ptSamples 4.  The strongly chromatic medium runs past 64 scatters per path; a
device error (B200PT_E_DEVICE) would raise from render_headless."""
import numpy as np
import pytest

import estcases
import volcases as VC
from vk_gltf_renderer_b200.renderer import PathTracer, Resources, render_headless

pytestmark = pytest.mark.gpu

W = H = 288


def _render(case, frames, max_depth=5, spp=1, batch=1):
    scn = VC.scene(case)
    res = Resources(scene=scn, hdr_rgb=VC.env_rgb(case), camera=scn.camera, size=(W, H))
    res.settings.hdrEnvRotation = case.get("rotation", 0.0)
    res.settings.hdrEnvIntensity = case.get("intensity", 1.0)
    pt = PathTracer(0)
    pt.ptMaxDepth, pt.ptSamples, pt.ptFireflyClamp = max_depth, spp, estcases.NO_CLAMP
    pt.onAttach(res)
    pt.set_frame_batch(batch)
    pt, img = render_headless(res, frames, pt=pt)
    ids, _ = pt.read_selection()
    pt.onDetach()
    estcases.assert_no_clamp(img, frames, spp)
    return img, VC.mask(ids)


@pytest.mark.parametrize("name", sorted(VC.ABSORB1))
def test_gpu_absorber_ior1(oracle_mod, name):
    case = VC.ABSORB1[name]
    img, m = _render(case, 2)
    E = VC.absorber_E(case, VC.environment(oracle_mod, case))
    report = []
    if case.get("mean"):
        ok, ok_sens = estcases.check_face(img, m, E, f"absorber {name} (face mean)", report)
        ok = ok and ok_sens
    else:
        ok = VC.check_pixels(img, m, E, f"absorber {name}", report)
    print(report[0])
    assert m.sum() > 50000
    assert ok, report[0]


@pytest.mark.parametrize("batch", [1, 3])
@pytest.mark.parametrize("name", sorted(VC.ABSORB15))
def test_gpu_absorber_ior15(oracle_mod, name, batch):
    case = VC.ABSORB15[name]
    spp = case["spp"]
    img, m = _render(case, (160 if case["max_depth"] == 2 else 12) // spp, max_depth=case["max_depth"], spp=spp, batch=batch)
    E = VC.absorber_E(case, VC.environment(oracle_mod, case))
    if not E.any():
        assert np.abs(img[m][:, :3]).mean() < 1e-5
        return
    report = []
    ok_val, ok_sens = estcases.check_face(img, m, E, f"absorber ior 1.5 {name} batch {batch}", report)
    print(report[0])
    assert ok_val, report[0]
    assert ok_sens, report[0]


@pytest.mark.parametrize("name", sorted(VC.SCATTER))
def test_gpu_scattering(oracle_mod, name):
    case = VC.SCATTER[name]
    img, m = _render(case, 40 * case.get("frames", 1), max_depth=case.get("max_depth", 12))
    if case.get("loose"):
        # no mean to compare (volcases.SCATTER): the walk ran past 64 scatters to the end, no device error, finite image
        print(f"scattering {name}: face mean {img[m][:, :3].astype(np.float64).mean(0)}")
        return
    E, se = VC.scatter_E(oracle_mod, name)
    report = []
    ok_val, ok_sens = VC.check_mc(img, m, E, se, f"scattering {name}", report)
    print(report[0])
    assert ok_val, report[0]
    assert ok_sens, report[0]


@pytest.mark.parametrize("batch,spp", [(3, 1), (1, 4)])
def test_gpu_scattering_batch_spp(oracle_mod, batch, spp):
    name = "grey_g0.3_tau3.0"
    case = VC.SCATTER[name]
    img, m = _render(case, 40 // spp, max_depth=12, spp=spp, batch=batch)
    E, se = VC.scatter_E(oracle_mod, name)
    report = []
    ok_val, ok_sens = VC.check_mc(img, m, E, se, f"scattering {name} batch {batch} spp {spp}", report)
    print(report[0])
    assert ok_val, report[0]
    assert ok_sens, report[0]
