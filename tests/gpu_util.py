"""Helpers shared by the -m gpu tests: device buffers through torch (plumbing only)."""
import numpy as np


def to_dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def primary_rays(cam, w, h, jitter=0.5):
    """Pinhole camera rays (o,tmin,d,tmax) for ray-level parity tests."""
    from vk_gltf_renderer_b200 import camera as cm
    import math
    view = cm.look_at(cam.eye, cam.center, cam.up)
    vinv = np.linalg.inv(view)
    t = math.tan(cam.yfov / 2)
    xs, ys = np.meshgrid(np.arange(w), np.arange(h))
    cx = ((xs + jitter) / w * 2 - 1) * t * (w / h)
    cy = -((ys + jitter) / h * 2 - 1) * t
    d = np.stack([cx, cy, -np.ones_like(cx)], -1).reshape(-1, 3)
    d = d @ vinv[:3, :3].T
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    rays = np.zeros((w * h, 8), np.float32)
    rays[:, 0:3] = vinv[:3, 3]
    rays[:, 3] = 0.0
    rays[:, 4:7] = d
    rays[:, 7] = 1e32
    return rays


def random_rays(n, lo, hi, seed=1234):
    rng = np.random.default_rng(seed)
    lo, hi = np.asarray(lo, np.float64), np.asarray(hi, np.float64)
    c, r = (lo + hi) / 2, np.linalg.norm(hi - lo) / 2
    o = c + rng.normal(size=(n, 3)) * r
    tgt = c + (rng.random((n, 3)) - 0.5) * (hi - lo)
    d = tgt - o
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    rays = np.zeros((n, 8), np.float32)
    rays[:, 0:3] = o
    rays[:, 4:7] = d
    rays[:, 7] = 1e32
    return rays


def trace_both(pt, o, rays, seeds, tmax=4.0, float_cols=()):
    """Closest-hit rays, then the same rays as shadow rays cut at tmax, through the device's ray-level API and the oracle.
    The hits must be equal bit for bit, except the columns in float_cols, which are compared as floats.  The seeds and the
    shadow transmission must be exact.  Returns the oracle's hits, seeds, transmission and shadow-ray seeds."""
    import torch
    s_ref = seeds.copy()
    ref = o.trace_closest(rays, s_ref)
    d_rays, d_seeds = to_dev(rays), to_dev(seeds.copy())
    d_hits = torch.empty((len(rays), 6), dtype=torch.float32, device="cuda")
    pt.trace_closest(d_rays.data_ptr(), len(rays), d_hits.data_ptr(), d_seeds.data_ptr())
    pt.synchronize()
    got = d_hits.cpu().numpy()
    bits = [c for c in range(got.shape[1]) if c not in float_cols]
    assert np.array_equal(got.view(np.uint32)[:, bits], ref.view(np.uint32)[:, bits])
    assert np.array_equal(got[:, list(float_cols)], ref[:, list(float_cols)])
    assert np.array_equal(d_seeds.cpu().numpy(), s_ref)
    rays_s = rays.copy()
    rays_s[:, 7] = tmax
    ss_ref = seeds.copy()
    ref_t = o.trace_shadow(rays_s, ss_ref)
    d_rays, d_seeds = to_dev(rays_s), to_dev(seeds.copy())
    d_t = torch.empty((len(rays), 3), dtype=torch.float32, device="cuda")
    pt.trace_shadow(d_rays.data_ptr(), len(rays), d_t.data_ptr(), d_seeds.data_ptr())
    pt.synchronize()
    assert np.array_equal(d_t.cpu().numpy(), ref_t)
    assert np.array_equal(d_seeds.cpu().numpy(), ss_ref)
    return ref, s_ref, ref_t, ss_ref
