"""The device's images converge to the float64 expectation of the estimator (tests/estref.py): the cases of
test_estimator_expectation.py at a larger image, rendered through render_headless.  The alias table of the expectation is
the one the CPU oracle builds from the same environment."""
import numpy as np
import pytest

import estcases as C
import estref
from vk_gltf_renderer_b200 import synth
from vk_gltf_renderer_b200.renderer import PathTracer, Resources, render_headless

pytestmark = pytest.mark.gpu

W = H = 288


def _render(scn, env_rgb, case, w, h, frames, max_depth=5, spp=1, batch=1):
    res = Resources(scene=scn, hdr_rgb=env_rgb, camera=scn.camera, size=(w, h))
    res.settings.hdrEnvRotation = case.get("rotation", 0.0)
    res.settings.hdrEnvIntensity = case.get("intensity", 1.0)
    pt = PathTracer(0)
    pt.ptMaxDepth, pt.ptSamples, pt.ptFireflyClamp = max_depth, spp, C.NO_CLAMP
    pt.onAttach(res)
    pt.set_frame_batch(batch)
    pt, img = render_headless(res, frames, pt=pt)
    ids, _ = pt.read_selection()
    pt.onDetach()
    C.assert_no_clamp(img, frames, spp)
    return img, ids


@pytest.mark.parametrize("name", sorted(C.POLY_CASES))
def test_gpu_polyhedron_faces(oracle_mod, name):
    case = C.POLY_CASES[name]
    scn, normals = C.poly_scene(case)
    env_rgb = C.env_rgb(case)
    img, ids = _render(scn, env_rgb, case, W, H, max(16, case["frames"] // 2))
    o = oracle_mod.Oracle()
    o.set_environment(env_rgb)
    env = estref.Env.from_oracle(o)
    faces = C.face_masks(ids, 2500)
    assert len(faces) >= 4, "too few faces large enough to test"
    report, bad, insensitive = [], [], []
    for k, m in faces.items():
        E = C.expected_face(case, env, scn, normals, k, m, W, H)
        ok_val, ok_sens = C.check_face(img, m, E, f"{name} face {k}", report)
        bad += [] if ok_val else [k]
        insensitive += [] if ok_sens else [k]
    print("\n".join(report))
    assert not bad, f"faces {bad} off their expectation:\n" + "\n".join(report)
    assert not insensitive, f"faces {insensitive} too noisy to see a 1 % bias:\n" + "\n".join(report)


@pytest.mark.parametrize("batch", [1, 3])
@pytest.mark.parametrize("rho,depth,spp", C.ENCLOSURE_CASES)
def test_gpu_enclosure(rho, depth, spp, batch):
    scn = synth.synth_enclosure(rho, C.ENCLOSURE_E)
    w = h = 96
    img, _ = _render(scn, C.furnace_env(), dict(intensity=0.0), w, h, 48 // spp, max_depth=depth, spp=spp, batch=batch)
    E = estref.enclosure_expectation(C.ENCLOSURE_E, rho, depth)
    report = []
    ok_val, ok_sens = C.check_face(img, np.ones((h, w), bool), E, f"enclosure rho={rho} depth={depth} spp={spp} batch={batch}", report)
    print(report[0])
    assert ok_val, report[0]
    assert ok_sens, report[0]
