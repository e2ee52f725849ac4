"""The per-pixel convergence rule (csrc/converge.cuh, what k_accumulate<true> runs) compiled for the host
(tools/host_converge_check.cpp) on synthetic frame streams, against the float64 two-pass restatement of tests/convref.py:
M2 within a first-order fp32 bound, the stop decisions equal except where e lies within that bound's margin of the threshold, and
stops only at checkpoints, never before minFrames."""
import os
import subprocess
import zlib

import numpy as np
import pytest

import convref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "vk_gltf_renderer_b200", "csrc")
CUDA_INC = os.environ.get("CUDA_HOME", "/usr/local/cuda") + "/include"


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    if not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")):
        pytest.skip("CUDA headers not found")
    path = str(tmp_path_factory.mktemp("conv") / "host_converge_check")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-I" + CUDA_INC, "-o", path,
                           os.path.join(CSRC, "tools", "host_converge_check.cpp")])
    return path


def run(exe, tmp, sums, ns, threshold, floor, min_frames, interval):
    F, P = sums.shape[:2]
    with open(tmp / "in.bin", "wb") as f:
        f.write(np.array([P, F], np.uint32).tobytes())
        f.write(np.array([threshold, floor], np.float32).tobytes())
        f.write(np.array([min_frames, interval], np.uint32).tobytes())
        for k in range(F):
            f.write(np.int32(ns[k]).tobytes())
            f.write(np.ascontiguousarray(sums[k], np.float32).tobytes())
    subprocess.check_call([exe, str(tmp / "in.bin"), str(tmp / "out.bin")])
    raw = np.fromfile(str(tmp / "out.bin"), np.uint32)
    stop = raw[:P]
    per = raw[P:].view(np.float32).reshape(F, 2, P)
    return stop, per[:, 0].astype(np.float64), per[:, 1].astype(np.float64)


STREAMS = {
    "1spp": lambda rng, F: np.ones(F, np.int64),
    "3spp": lambda rng, F: np.full(F, 3, np.int64),
    "varying": lambda rng, F: rng.integers(1, 9, F),
}


@pytest.mark.parametrize("frames,threshold,interval", [(256, 0.05, 8), (1024, 0.01, 4), (4096, 0.003, 16)])
@pytest.mark.parametrize("spp", sorted(STREAMS))
def test_rule_against_float64(exe, tmp_path, spp, frames, threshold, interval):
    rng = np.random.default_rng(zlib.crc32(f"{spp}{frames}".encode()))
    kinds = R.pixel_kinds(rng, 6 if frames <= 1024 else 2)
    ns = STREAMS[spp](rng, frames)
    sums = R.stream(rng, kinds, ns)
    floor, min_frames = 1e-3, 16
    stop, m2, e = run(exe, tmp_path, sums, ns, threshold, floor, min_frames, interval)
    P = sums.shape[1]

    # stops only at checkpoints, never before minFrames
    s = stop[stop > 0].astype(np.int64)
    assert (s % interval == 0).all() and (s >= min_frames).all()
    # a stopped pixel's recorded values end at its stop frame
    for p in np.nonzero(stop)[0][:8]:
        assert np.isnan(m2[stop[p]:, p]).all() and not np.isnan(m2[stop[p] - 1, p])

    # flat and black pixels included, e is never NaN with floor > 0 (M2 is clamped at 0 where rounding takes it below)
    assert not np.isnan(e[np.isfinite(m2)]).any()

    c = R.lum(R.frame_means(sums, ns))
    bound = R.m2_bound(c, ns)
    N = np.cumsum(ns)
    near = 0
    decided = np.zeros(P, bool)  # the pixel's 64-bit history left the fp32 one (a decision inside the margin): no further compare
    for F in range(interval, frames + 1, interval):
        live = (stop == 0) | (stop >= F)
        live &= ~decided
        m64, m2_64 = R.two_pass(c, ns, F)
        got = m2[F - 1]
        assert np.all(np.abs(got[live] - m2_64[live]) <= bound[F - 1][live] + 1e-300), F
        if F < min_frames:
            assert not (stop == F).any()
            continue
        e64 = R.rel_error(m2_64, F, N[F - 1], m64, floor)
        # margin: e over M2 +- bound and the mean's fp32 uncertainty
        eps_m = 4 * R.U * F * np.abs(c[:F]).max(0) + 2 * R.U * np.abs(m64)
        lo = R.rel_error(np.maximum(m2_64 - bound[F - 1], 0), F, N[F - 1], m64 + eps_m, floor) * (1 - 1e-6)
        hi = R.rel_error(m2_64 + bound[F - 1], F, N[F - 1], np.maximum(m64 - eps_m, 0), floor) * (1 + 1e-6)
        stop32 = stop == F
        stop64 = e64 <= threshold
        differ = live & (stop32 != stop64)
        inside = (lo <= threshold) & (threshold <= hi)
        assert not (differ & ~inside).any(), (F, np.nonzero(differ & ~inside))
        near += int((differ).sum())
        decided |= differ
        # e as the host check reports it is the fp32 value whose comparison made the decision
        assert np.array_equal(e[F - 1][live & stop32] <= threshold, np.ones(int((live & stop32).sum()), bool))
    print(f"\n{spp} F={frames}: {int((stop > 0).sum())}/{P} stopped at {len(np.unique(stop[stop > 0]))} checkpoints; "
          f"{near} decisions within the fp32 margin of the threshold")
    assert near <= max(2, P // 50)
