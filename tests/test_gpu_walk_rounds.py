"""-m gpu: the any-hit continuation rounds of a bounce's walks (B200PT_CONT_ROUNDS) and the grids of the rounds after the first
(B200PT_CONT_SMALL_GRID) change where the walk sequence walk -> [k_alpha -> continuation walk] x R -> k_alpha splits its work, never
what it computes.  The ray-level API runs that sequence, so its hits, seeds and transmission are bit-exact against the oracle for every
round count; frames render the same image; and the launch counts follow the sequence.  Both knobs are read when a handle is created."""
import functools

import numpy as np
import pytest

from gpu_util import random_rays, to_dev, trace_both
from test_gpu_omm import deep_layers_with_micromaps
from test_gpu_scenes import _attach

pytestmark = pytest.mark.gpu

ROUNDS = (1, 2, 8)


@functools.lru_cache(maxsize=None)
def _ray_case(name):
    from vk_gltf_renderer_b200 import synth
    if name == "sampler_layers":
        # 14 alpha layers: rays through all of them reach the in-kernel fallback of the last k_alpha at R = 1 and R = 2
        rays = random_rays(60000, [-1.6, 0.1, -2.2], [1.9, 2.1, 0.2])
        seeds = ((np.arange(len(rays), dtype=np.uint64) * 2654435761) % (2 ** 32)).astype(np.uint32)
        return synth.sampler_layers(), rays, seeds, 4.0
    scn, _, rays, seeds = deep_layers_with_micromaps()
    return scn, rays, seeds, 0.7


def _launches_per_call(pt, rays):
    """kernelLaunches of one trace_closest and one trace_shadow call"""
    import torch
    d_rays = to_dev(rays)
    d_out = torch.empty((len(rays), 6), dtype=torch.float32, device="cuda")
    out = []
    for call in (pt.trace_closest, pt.trace_shadow):
        k0 = pt.stats()["kernelLaunches"]
        call(d_rays.data_ptr(), len(rays), d_out.data_ptr())
        out.append(pt.stats()["kernelLaunches"] - k0)
    pt.synchronize()
    return out


@pytest.mark.parametrize("small_grid", [0, 1])
@pytest.mark.parametrize("rounds", ROUNDS)
@pytest.mark.parametrize("case", ["sampler_layers", "layers_micromaps"])
def test_ray_level_results_do_not_depend_on_the_rounds(std_env, oracle_mod, monkeypatch, case, rounds, small_grid):
    monkeypatch.setenv("B200PT_CONT_ROUNDS", str(rounds))
    monkeypatch.setenv("B200PT_CONT_SMALL_GRID", str(small_grid))
    scn, rays, seeds, tmax = _ray_case(case)
    pt, _ = _attach(scn, std_env, (16, 16))
    o = oracle_mod.Oracle()
    o.set_scene(scn)
    trace_both(pt, o, rays, seeds, tmax=tmax)
    assert _launches_per_call(pt, rays) == [4 + 2 * rounds] * 2
    pt.onDetach()


@pytest.mark.parametrize("rounds", ROUNDS)
def test_ray_level_launches_without_non_opaque_triangles(std_env, box_scene, monkeypatch, rounds):
    monkeypatch.setenv("B200PT_CONT_ROUNDS", str(rounds))
    pt, _ = _attach(box_scene, std_env, (16, 16))
    lo, hi = box_scene.bounds()
    assert _launches_per_call(pt, random_rays(1000, lo, hi)) == [3, 3]
    pt.onDetach()


def _render_three_frames(scn, env, depth, rounds, monkeypatch):
    """frames 0..2 at one sample: the second frame's launches, the third one's profiled per-stage launches, the image and the ray
    counters"""
    monkeypatch.setenv("B200PT_CONT_ROUNDS", str(rounds))
    pt, res = _attach(scn, env, (200, 120), ptMaxDepth=depth, ptSamples=1)
    res.frameCount = 0
    pt.onRender(None, res)
    k0 = pt.stats()["kernelLaunches"]
    res.frameCount = 1
    pt.onRender(None, res)
    second = pt.stats()["kernelLaunches"] - k0
    counters = {k: pt.stats()[k] for k in ("closestRays", "shadowRays", "shadedHits", "pathsStarted")}
    pt.set_profiling(True)
    pt.reset_stats()
    res.frameCount = 2
    pt.onRender(None, res)
    third = pt.stats()
    img = pt.read_accum()
    pt.onDetach()
    return second, third, img, counters


def test_frames_do_not_depend_on_the_rounds(std_env, monkeypatch):
    """SynthSponza-small (MASK foliage, no volume) at one sample and depth 5: image and ray counters bit-identical for R = 1, 2, 8,
    2 + depth x (6 + 4R) launches per frame, and per frame depth x (1 + R) closest walks, as many shadow walks and depth x (2 + 2R)
    any-hit launches"""
    from vk_gltf_renderer_b200 import synth
    scn = synth.synth_sponza(tex_size=128, detail=0.05)
    depth = 5
    runs = {r: _render_three_frames(scn, std_env, depth, r, monkeypatch) for r in ROUNDS}
    _, _, img1, counters1 = runs[1]
    assert counters1["shadedHits"] > 0 and (img1[..., :3] > 0).any()
    for r, (second, third, img, counters) in runs.items():
        assert np.array_equal(img.view(np.uint32), img1.view(np.uint32)), r
        assert counters == counters1, r
        assert second == 2 + depth * (6 + 4 * r)
        assert third["kernelLaunches"] == second
        assert third["launchesTraceClosest"] == depth * (1 + r) and third["launchesTraceShadow"] == depth * (1 + r)
        assert third["launchesAnyHit"] == depth * (2 + 2 * r)
