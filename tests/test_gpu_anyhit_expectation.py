"""-m gpu: the device's any-hit sequence (k_trace / k_shadow -> k_alpha -> continuation rounds -> k_alpha and its in-kernel
fallback walks), run by trace_closest / trace_shadow with seeds, against the float64 model of anyhitref.py: per ray against the
replay of its draws, and in distribution against the order-free probabilities (anyhitcases.py).  Every case runs with the
default switches; the deep ones also with 1, 2 and 8 continuation rounds (B200PT_CONT_ROUNDS), the device tree builder, and
without alpha caps (B200PT_ALPHA_CAPS=0); the MASK layers once more with opacity micromaps baked into the scene.  Rendered
frames run the same stage from the bounce loop: emissive veils in front of the camera and shadow veils between a light and a
lit body converge to their float64 expectations (estcases' statistics, the firefly clamp off)."""
import numpy as np
import pytest

import anyhitcases as hc
from gpu_util import to_dev
from test_gpu_scenes import _attach

pytestmark = pytest.mark.gpu

ALL_CASES = [f"veils-{n}-{s}" for n in hc.VEIL_COUNTS for s in ("1s", "2s")] + ["ties", "textured", "mirrored", "mask", "occluded",
                                                                                 "tinted"]
DEEP_CASES = ["veils-13-1s", "veils-29-2s", "veils-45-2s", "ties", "textured", "mirrored", "mask", "occluded", "tinted"]
CONFIGS = {"rounds1": dict(rounds=1), "rounds2": dict(rounds=2), "rounds8": dict(rounds=8), "device_bvh": dict(builder=1),
           "no_caps": dict(caps=0)}


def _device(scn, std_env, monkeypatch, rounds=None, builder=0, caps=None):
    if rounds is not None:
        monkeypatch.setenv("B200PT_CONT_ROUNDS", str(rounds))
    if caps is not None:
        monkeypatch.setenv("B200PT_ALPHA_CAPS", str(caps))
    pt, res = _attach(scn, std_env, (16, 16))
    if builder:
        pt.set_bvh_builder(builder)
        pt.onSceneInvalidated(res)
    return pt


def _trace(pt, rays, seeds, shadow):
    import torch
    d_rays, d_seeds = to_dev(rays), to_dev(seeds.copy())
    out = torch.empty((len(rays), 3 if shadow else 6), dtype=torch.float32, device="cuda")
    (pt.trace_shadow if shadow else pt.trace_closest)(d_rays.data_ptr(), len(rays), out.data_ptr(), d_seeds.data_ptr())
    pt.synchronize()
    return out.cpu().numpy(), d_seeds.cpu().numpy()


def _run(c, pt, count_draws=True, rows=None):
    report = []
    rows = np.arange(len(c.rays)) if rows is None else rows
    if c.closest is not None:
        hits, seeds = _trace(pt, c.rays[rows], c.closest["seeds"][rows], False)
        hc.check_closest(c, hits, seeds, report, count_draws, rows=rows)
        hc.check_closest_distribution(c, hits, seeds, report, count_draws, rows=rows)
    T, seeds = _trace(pt, c.rays_s[rows], c.shadow["seeds"][rows], True)
    hc.check_shadow(c, T, seeds, report, count_draws, rows=rows)
    hc.check_shadow_distribution(c, T, seeds, report, count_draws, rows=rows)
    print("\n".join(report))


@pytest.mark.parametrize("name", ALL_CASES)
def test_device_matches_the_replay_and_the_expectation(std_env, monkeypatch, name):
    c = hc.case(name)
    pt = _device(c.scn, std_env, monkeypatch)
    _run(c, pt)
    pt.onDetach()


@pytest.mark.parametrize("config", list(CONFIGS))
@pytest.mark.parametrize("name", DEEP_CASES)
def test_device_switches_change_nothing_the_model_sees(std_env, monkeypatch, name, config):
    c = hc.case(name)
    pt = _device(c.scn, std_env, monkeypatch, **CONFIGS[config])
    _run(c, pt)
    pt.onDetach()


@pytest.mark.parametrize("count", [1, 31, 4097])
def test_device_partial_warps(std_env, monkeypatch, count):
    """k_alpha runs 8 paths per warp: 1, 31 and 4097 rays leave partial warps in every round"""
    c = hc.case("veils-13-2s")
    pt = _device(c.scn, std_env, monkeypatch)
    _run(c, pt, rows=np.arange(count))
    pt.onDetach()


def test_device_mask_layers_with_micromaps(std_env, monkeypatch):
    """the MASK layers with level-3 micromaps: resolved micro-triangles draw nothing, so the hits and the transmission are
    compared with the replay and the distributions, and the draw counts are not; the rays whose first draw was chosen to land
    on a transparent texel (accepted without micromaps) are left out of both"""
    from vk_gltf_renderer_b200 import omm, synth
    c = hc.case("mask")
    scn = synth.synth_layers()
    st = omm.bake_opacity_micromaps(scn, level=3)
    assert st["opaque"] > 0 and st["transparent"] > 0
    pt = _device(scn, std_env, monkeypatch)
    rows = np.nonzero(~c.closest["edge"] & ~c.shadow["edge"])[0]
    _run(c, pt, count_draws=False, rows=rows)
    pt.onDetach()


# ---- the frame path: the bounce loop's k_trace / k_shadow queues into k_alpha, per-bounce seeds, NEE shadow rays ---------------
@pytest.mark.parametrize("batch", [1, 3])
@pytest.mark.parametrize("n", hc.EMISSIVE_VEIL_COUNTS)
def test_device_emissive_veils(n, batch):
    """black BLEND layers with distinct emission in front of a constant environment, rendered (frame batch 1 and 3): every
    pixel converges to sum_i e_i p_i prod_{j<i} (1 - p_j) + L prod_j (1 - p_j), p on the closest-hit grid"""
    import estcases as C
    from test_gpu_estimator_expectation import _render
    scn, E = hc.emissive_veils(n, C.FURNACE_L)
    w = h = 128
    img, _ = _render(scn, C.furnace_env(), {}, w, h, 24, max_depth=2, batch=batch)
    report = []
    ok_val, ok_sens = C.check_face(img, np.ones((h, w), bool), E, f"emissive veils n={n} batch={batch}", report)
    print(report[0])
    assert ok_val and ok_sens, report[0]


@pytest.mark.parametrize("n", hc.SHADOW_VEIL_COUNTS)
def test_device_shadow_veils(oracle_mod, n):
    """the light-only faces of the furnace polyhedron behind n black BLEND layers (every other one single-sided, facing away
    from the body; one of alpha 0 from n = 5): each face converges to its light-only expectation times prod_i (1 - p_i), p on
    the shadow grid"""
    import estcases as C
    import estref
    from test_gpu_estimator_expectation import _render
    scn, normals, case, factor = hc.shadow_veils(n)
    assert hc.veils_off_view(scn, 20) > 1.0
    w = h = 288
    img, ids = _render(scn, C.furnace_env(), case, w, h, 100)
    o = oracle_mod.Oracle()
    o.set_environment(C.furnace_env())
    env = estref.Env.from_oracle(o)
    faces = C.face_masks(ids, 2500)
    assert len(faces) >= 4
    report, bad, lit = [], [], 0
    for k, m in faces.items():
        E = C.expected_face(case, env, scn, normals, k, m, w, h) * factor
        lit += int(np.max(E) > 0)
        ok_val, ok_sens = C.check_face(img, m, E, f"shadow veils n={n} face {k}", report)
        bad += [] if (ok_val and ok_sens) else [k]
    print("\n".join(report))
    assert lit >= 2, "too few lit faces"
    assert not bad, "\n".join(report)
