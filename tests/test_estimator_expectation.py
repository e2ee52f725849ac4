"""The CPU oracle's images converge to the float64 expectation of the estimator (tests/estref.py): white furnace, GGX furnace,
environment-lit and light-lit faces of a convex icosahedron, and a closed emissive enclosure.  See tests/estcases.py for the
statistics.  The device runs the same cases in test_gpu_estimator_expectation.py."""
import numpy as np
import pytest

import estcases as C
import estref
from vk_gltf_renderer_b200 import camera as camm
from vk_gltf_renderer_b200 import synth

W = H = 192


def _render(O, scn, env, fi, w, h, frames, max_depth=5, spp=1):
    o = O.Oracle()
    o.set_scene(scn)
    o.set_environment(env)
    acc = np.zeros((h, w, 4), np.float32)
    ids = np.zeros((h, w), np.uint32)
    for f in range(frames):
        pc = camm.make_push_constant(scn.camera, h, frame_count=f, total_samples=f * spp, num_samples=spp, max_depth=max_depth,
                                     firefly_clamp=C.NO_CLAMP)
        o.render_frame(fi, pc, acc, object_id=ids if f == 0 else None)
    C.assert_no_clamp(acc, frames, spp)
    return acc, ids, o


@pytest.mark.parametrize("name", sorted(C.POLY_CASES))
def test_polyhedron_faces(oracle_mod, name):
    case = C.POLY_CASES[name]
    scn, normals = C.poly_scene(case)
    env_rgb = C.env_rgb(case)
    acc, ids, o = _render(oracle_mod, scn, env_rgb, C.frame_info(scn, W, H, case), W, H, case["frames"])
    env = estref.Env.from_oracle(o)
    faces = C.face_masks(ids, 500)
    assert len(faces) >= 4, "too few faces large enough to test"
    report, bad, insensitive = [], [], []
    for k, m in faces.items():
        E = C.expected_face(case, env, scn, normals, k, m, W, H)
        ok_val, ok_sens = C.check_face(acc, m, E, f"{name} face {k}", report)
        bad += [] if ok_val else [k]
        insensitive += [] if ok_sens else [k]
    print("\n".join(report))
    assert not bad, f"faces {bad} off their expectation:\n" + "\n".join(report)
    assert not insensitive, f"faces {insensitive} too noisy to see a 1 % bias:\n" + "\n".join(report)


@pytest.mark.parametrize("rho,depth,spp", C.ENCLOSURE_CASES)
def test_enclosure(oracle_mod, rho, depth, spp):
    scn = synth.synth_enclosure(rho, C.ENCLOSURE_E)
    env = C.furnace_env()
    w = h = 48
    fi = camm.make_frame_info(scn.camera, w, h, env_intensity=0.0)
    frames = 40 // spp
    acc, _, _ = _render(oracle_mod, scn, env, fi, w, h, frames, max_depth=depth, spp=spp)
    E = estref.enclosure_expectation(C.ENCLOSURE_E, rho, depth)
    report = []
    ok_val, ok_sens = C.check_face(acc, np.ones((h, w), bool), E, f"enclosure rho={rho} depth={depth} spp={spp}", report)
    print(report[0])
    assert ok_val, report[0]
    assert ok_sens, report[0]
