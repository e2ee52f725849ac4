"""GPU: b200pt_set_convergence stops each pixel of an accumulation once its relative error is below the threshold.  A pixel that
stopped after frame F must be bit-identical to the plain render's pixel after frame F - 1 (and a pixel that never stopped to the plain
render's last image); images, stop frames and errors must not depend on frames in flight, frame batching, tiles or bands; the ray
counters must count only the paths of active pixels."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

W, H = 64, 48
DEPTH = 6
E_INVALID, E_UNSUPPORTED = -1, -4
SPP = {"1spp": lambda f: 1, "3spp": lambda f: 3, "varying": lambda f: (1, 3, 2, 4, 1, 2)[f % 6]}


@pytest.fixture(scope="module")
def scenes():
    from vk_gltf_renderer_b200 import synth
    return {"sponza_plane": synth.synth_sponza(tex_size=128, detail=0.05), "glass_volume": synth.synth_glass(scatter=True),
            "lit": synth.synth_lit()}


def _tracer(scn, env, lanes=1, batch=1, tile=None):
    from vk_gltf_renderer_b200.renderer import PathTracer, Resources
    res = Resources(scene=scn, hdr_rgb=env, camera=scn.camera, size=(W, H), tile=tile)
    pt = PathTracer(0)
    pt.onAttach(res)
    pt.set_frames_in_flight(lanes)
    pt.set_frame_batch(batch)
    return pt


def _frames(scn, n, spp, plane):
    from vk_gltf_renderer_b200 import camera
    fi = camera.make_frame_info(scn.camera, W, H, infinite_plane=plane, plane_distance=-0.05, shadow_catcher=False)
    pcs, total = [], 0
    for f in range(n):
        s = SPP[spp](f)
        pcs.append(camera.make_push_constant(scn.camera, H, frame_count=f, total_samples=total, num_samples=s, max_depth=DEPTH))
        total += s
    return fi, pcs


def _render(pt, fi, pcs, conv=None):
    """conv = (threshold, minFrames, interval): (image, selection, stop, error, pathsStarted)"""
    if conv:
        pt.set_convergence(conv[0], floor=1e-3, min_frames=conv[1], interval=conv[2])
    pt.reset_stats()
    for pc in pcs:
        pt.render_frame_raw(fi, pc)
    img = pt.read_accum()
    sel = pt.read_selection()
    stop, err, _ = pt.read_convergence() if conv else (None, None, None)
    return img, sel, stop, err, pt.stats()["pathsStarted"]


def _snapshots(pt, fi, pcs):
    snaps = []
    for pc in pcs:
        pt.render_frame_raw(fi, pc)
        snaps.append(pt.read_accum())
    return np.stack(snaps), pt.read_selection()


def _pick_threshold(pt, fi, pcs, min_frames, interval):
    """the largest threshold of a sweep at which pixels stop at three or more checkpoints and some never stop"""
    for thr in (0.5, 0.3, 0.2, 0.1, 0.05, 0.03, 0.02, 0.01, 0.005):
        r = _render(pt, fi, pcs, (thr, min_frames, interval))
        stop = r[2]
        if len(np.unique(stop[stop > 0])) >= 3 and (stop == 0).any():
            return thr, r
    raise AssertionError("no threshold of the sweep stops pixels at three checkpoints and leaves some active")


@pytest.mark.parametrize("spp", sorted(SPP))
@pytest.mark.parametrize("scene", ["sponza_plane", "glass_volume", "lit"])
def test_stopped_pixels_equal_the_plain_render_at_their_stop_frame(scenes, std_env, scene, spp):
    scn = scenes[scene]
    fi, pcs = _frames(scn, 48, spp, scene == "sponza_plane")
    plain = _tracer(scn, std_env)
    snaps, sel = _snapshots(plain, fi, pcs)
    plain.onDetach()
    pt = _tracer(scn, std_env)
    thr, (img, csel, stop, err, started) = _pick_threshold(pt, fi, pcs, 8, 4)
    idx = np.where(stop > 0, stop.astype(np.int64) - 1, len(pcs) - 1)
    want = np.take_along_axis(snaps, idx[None, :, :, None], 0)[0]
    assert np.array_equal(img.view(np.uint32), want.view(np.uint32))
    assert np.array_equal(csel[0], sel[0]) and np.array_equal(csel[1].view(np.uint32), sel[1].view(np.uint32))
    # the read-back: stopped pixels at checkpoints past minFrames with e <= threshold, active ones above it after the last checkpoint
    s = stop[stop > 0]
    assert (s % 4 == 0).all() and (s >= 8).all()
    assert (err[stop > 0] <= np.float32(thr)).all() and (err[stop == 0] > np.float32(thr)).all()
    # counters: numSamples x active pixels per frame
    active = [int(((stop == 0) | (stop > f)).sum()) for f in range(len(pcs))]
    assert started == sum(pc.numSamples * a for pc, a in zip(pcs, active))
    print(f"\n{scene} {spp}: threshold {thr}, {int((stop > 0).sum())}/{stop.size} stopped at checkpoints {sorted(set(s.tolist()))}")
    pt.onDetach()


@pytest.mark.parametrize("interval", [4, 6])
@pytest.mark.parametrize("lanes,batch,tile", [(4, 1, None), (1, 3, None), (4, 3, None), (1, 1, (8, 24)), (4, 3, (8, 24)),
                                              (1, 1, ("interleave", 4, 2, 1)), (4, 3, ("interleave", 4, 2, 1))])
def test_results_do_not_depend_on_scheduling(scenes, std_env, interval, lanes, batch, tile):
    scn = scenes["sponza_plane"]
    fi, pcs = _frames(scn, 36, "1spp", True)
    conv = (0.1, 8, interval)
    ref = _tracer(scn, std_env, tile=tile)
    a = _render(ref, fi, pcs, conv)
    ref.onDetach()
    pt = _tracer(scn, std_env, lanes, batch, tile)
    b = _render(pt, fi, pcs, conv)
    pt.onDetach()
    assert (a[2] > 0).any() and (a[2] == 0).any()
    for x, y in zip(a[:4], b[:4]):
        if isinstance(x, tuple):
            assert all(np.array_equal(u.view(np.uint32), v.view(np.uint32)) for u, v in zip(x, y))
        else:
            assert np.array_equal(x.view(np.uint32), y.view(np.uint32))
    assert a[4] == b[4]


def test_frames_after_every_pixel_stopped_change_nothing(scenes, std_env):
    scn = scenes["lit"]
    fi, pcs = _frames(scn, 40, "3spp", False)
    pt = _tracer(scn, std_env, lanes=4)
    img, _, stop, _, _ = _render(pt, fi, pcs[:16], (100.0, 8, 4))
    assert (stop == 8).all() and pt.read_convergence()[2] == 0
    pt.reset_stats()
    for pc in pcs[16:]:
        pt.render_frame_raw(fi, pc)
    assert np.array_equal(pt.read_accum().view(np.uint32), img.view(np.uint32))
    assert pt.stats()["pathsStarted"] == 0
    pt.onDetach()


def test_off_means_unchanged_and_settings_latch_at_a_first_frame(scenes, std_env):
    scn = scenes["sponza_plane"]
    fi, pcs = _frames(scn, 24, "1spp", True)
    fresh = _tracer(scn, std_env, lanes=4)
    want = _render(fresh, fi, pcs)
    fresh.onDetach()
    # on for one accumulation, then off: the next accumulation renders like a fresh handle
    pt = _tracer(scn, std_env, lanes=4)
    _render(pt, fi, pcs[:12], (0.2, 4, 4))
    pt.set_convergence(0)
    got = _render(pt, fi, pcs)
    assert np.array_equal(got[0].view(np.uint32), want[0].view(np.uint32)) and got[4] == want[4]
    assert pt._L.b200pt_read_convergence(pt._h, None, None, 0, None) == E_INVALID
    # a settings change in mid-accumulation does not alter that accumulation
    ref = _render(pt, fi, pcs, (0.1, 8, 4))
    pt.set_convergence(0.1, min_frames=8, interval=4)
    for k, pc in enumerate(pcs):
        if k == 10:
            pt.set_convergence(0.5, min_frames=2, interval=1)
        pt.render_frame_raw(fi, pc)
    stop, err, _ = pt.read_convergence()
    assert np.array_equal(pt.read_accum().view(np.uint32), ref[0].view(np.uint32)) and np.array_equal(stop, ref[2])
    assert np.array_equal(err.view(np.uint32), ref[3].view(np.uint32))
    pt.onDetach()


def test_refusals(scenes, std_env):
    from vk_gltf_renderer_b200 import abi
    scn = scenes["lit"]
    fi, pcs = _frames(scn, 2, "1spp", False)
    pt = _tracer(scn, std_env, lanes=2)
    L, h = pt._L, pt._h
    for bad in ((-0.1, 1e-3, 16, 8), (float("nan"), 1e-3, 16, 8), (0.1, -1.0, 16, 8), (0.1, float("nan"), 16, 8), (0.1, 1e-3, 1, 8),
                (0.1, 1e-3, 16, 0)):
        assert L.b200pt_set_convergence(h, C.byref(abi.Convergence(*bad))) == E_INVALID, bad
    assert L.b200pt_set_convergence(h, None) == 0
    pt.set_convergence(0.1, min_frames=4, interval=2)
    assert L.b200pt_set_views(h, 2) == E_UNSUPPORTED
    pt.set_guide_outputs(True)
    p = abi.PushConstant.from_buffer_copy(pcs[0])
    p.flags |= abi.PT_USE_OPTIX_DENOISER
    assert L.b200pt_render_frame(h, C.byref(fi), C.byref(p)) == E_UNSUPPORTED
    pt.set_guide_outputs(False)
    pt.set_dlss_guides(True)
    p = abi.PushConstant.from_buffer_copy(pcs[0])
    p.flags |= abi.PT_USE_DLSS
    assert L.b200pt_render_frame(h, C.byref(fi), C.byref(p)) == E_UNSUPPORTED
    pt.set_dlss_guides(False)
    pt.render_frame_raw(fi, pcs[0])
    pt.render_frame_raw(fi, pcs[1])
    # after a resize, the frame must start an accumulation
    from vk_gltf_renderer_b200.renderer import Resources
    pt.onResize(None, (W, H), Resources(size=(W, H)))
    assert L.b200pt_render_frame(h, C.byref(fi), C.byref(pcs[1])) == E_INVALID
    pt.render_frame_raw(fi, pcs[0])
    pt.set_convergence(0)
    pt.render_frame_raw(fi, pcs[0])
    pt.set_views(2)  # off again once latched off
    pt.onDetach()


def test_headless_ends_when_every_pixel_stopped(std_env, tmp_path):
    from vk_gltf_renderer_b200 import _lib, scene
    from vk_gltf_renderer_b200.renderer import PathTracer, Resources, render_headless
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    box = scene.load_gltf(os.path.join(root, "tests", "assets", "Box.glb"))
    exe = os.path.join(os.path.dirname(_lib.LIB_PATH), "b200pt_headless")
    blob, raw = str(tmp_path / "box.b2sc"), str(tmp_path / "box.raw")
    box.save_blob(blob, std_env)
    out = subprocess.run([exe, "--scene", blob, "--size", "96", "64", "--frames", "400", "--ptMaxDepth", "5", "--ptConvergenceThreshold", "0.05",
                          "--ptConvergenceMinFrames", "8", "--ptConvergenceInterval", "4", "--outRaw", raw], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr
    line = [l for l in out.stdout.splitlines() if l.startswith("HEADLESS_CONVERGED ")]
    assert len(line) == 1, out.stdout
    frames = int(line[0].split("frames=")[1].split(":")[0])
    assert frames < 400 and frames % 4 == 0
    img = np.fromfile(raw, np.float32).reshape(64, 96, 4)
    res = Resources(scene=box, hdr_rgb=std_env, camera=box.camera, size=(96, 64))
    pt = PathTracer(0)
    pt.ptMaxDepth = 5
    pt.onAttach(res)
    pt.set_convergence(0.05, min_frames=8, interval=4)
    pt, ref = render_headless(res, 400, pt=pt, until_converged=True)
    assert res.frameCount + 1 == frames
    # the two hosts compute the camera matrices independently (test_gpu_scenes.py): equal to rounding of the frame constants
    assert np.array_equal(img[..., 3], ref[..., 3])
    assert np.sqrt(np.mean((img[..., :3] - ref[..., :3]) ** 2)) <= 1e-4 * max(float(ref[..., :3].mean()), 1e-30)
    pt.onDetach()


def test_stopped_pixels_cover_the_known_expectation():
    """Coverage against ground truth: synth_furnace_polyhedron with Lambert rho 0.3 in the constant environment, whose faces have the
    float64 expectation E of tests/estref.py (estcases.expected_face).  Threshold 0.01, minFrames 16, interval 8, 32 spp per frame
    (frame means close to normal), at most 512 frames.  Most interior pixels must stop before the cap, and among stopped pixels the
    count with |v - E| > 4 threshold E must stay within a bound from the Student-t tail:
      with constant spp the frame means are i.i.d., and a pixel's (v - E) / (e v) is Student-t with F - 1 degrees of freedom at
      checkpoint F.  A pixel that stops at F has e <= threshold, so |v - E| > 4 threshold E means |t| > r / (threshold (1 + r)) with
      r = |v - E| / E > 4 threshold, i.e. |t| > 4 / (1 + 4 threshold).  Over the checkpoints, the expected number of such stops is at
      most sum_F (pixels active at F) x P(|t_{F-1}| > 4 / (1 + 4 threshold)); the count may exceed it by 4 binomial sigmas + 2.
    Reports the share and the mean signed deviation (v - E) / E of stopped pixels: the selection bias of data-dependent stopping (a
    pixel whose sample spread happens to be low stops early)."""
    from scipy import stats
    import estcases as EC
    from vk_gltf_renderer_b200.renderer import PathTracer, Resources, render_headless
    thr, min_frames, interval, cap, spp, size = 0.01, 16, 8, 512, 32, 192
    case = EC.FURNACE["furnace_lambert_0.3"]
    scn, normals = EC.poly_scene(case)
    res = Resources(scene=scn, hdr_rgb=EC.env_rgb(case), camera=scn.camera, size=(size, size))
    pt = PathTracer(0)
    pt.ptMaxDepth, pt.ptSamples, pt.ptFireflyClamp = 5, spp, EC.NO_CLAMP
    pt.onAttach(res)
    pt.set_convergence(thr, floor=1e-3, min_frames=min_frames, interval=interval)
    pt, img = render_headless(res, cap, pt=pt, until_converged=True)
    ids, _ = pt.read_selection()
    stop, err, _ = pt.read_convergence()
    pt.onDetach()
    faces = EC.face_masks(ids, 500)
    assert len(faces) >= 4, "too few faces large enough to test"
    v, E, st = [], [], []
    for k, m in faces.items():
        e_face = np.asarray(EC.expected_face(case, None, scn, normals, k, m, size, size), np.float64)
        v.append(img[m][:, :3].astype(np.float64).mean(-1))
        E.append(np.full(int(m.sum()), e_face.mean()))
        st.append(stop[m].astype(np.int64))
    v, E, st = np.concatenate(v), np.concatenate(E), np.concatenate(st)
    stopped = st > 0
    assert stopped.mean() > 0.5, f"only {stopped.mean():.3f} of the interior pixels stopped within {cap} frames"
    far = stopped & (np.abs(v - E) > 4 * thr * E)
    t_crit = 4.0 / (1.0 + 4.0 * thr)
    checkpoints = [F for F in range(interval, cap + 1, interval) if F >= min_frames]
    expect = sum(int(((st == 0) | (st >= F)).sum()) * 2.0 * stats.t.sf(t_crit, F - 1) for F in checkpoints)
    allowed = expect + 4.0 * np.sqrt(expect) + 2.0
    dev = (v - E) / E
    print(f"\nfurnace Lambert 0.3: {int(stopped.sum())}/{len(st)} interior pixels stopped (checkpoints {int(st[stopped].min())}.."
          f"{int(st[stopped].max())}); |v - E| > 4 threshold E: {int(far.sum())} = {far.sum() / stopped.sum():.5f} of the stopped "
          f"(bound {allowed:.1f} = {allowed / stopped.sum():.5f}); mean signed deviation of stopped pixels {dev[stopped].mean():+.5f}, "
          f"of all {dev.mean():+.5f}; mean e of stopped {err[stop > 0].mean():.5f}")
    assert far.sum() <= allowed
