"""The DEVICE traversal source on the host (-m "not gpu"): csrc/traverse.cuh is compiled by g++ through tools/host_shim.h (one
lane per warp) and checked against brute force by tools/host_traverse_check.cpp on the tree csrc/bvh.cpp builds -- the single-tree
closest walk (nearest opaque hit + the candidates in front of it, continuation walks resumed behind the last candidate and
refining the opaque hit) and the shadow walk (opaque occluder anywhere on the segment, else every candidate in order), with a
third and with seven eighths of the triangles flagged non-opaque.  This is the same node decode (PRMT plane bytes, conservative slack), compressed
stack and hit predicate the sm_90a kernels execute; what it cannot cover is warp-level scheduling."""
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "vk_gltf_renderer_b200", "csrc")
CUDA_INC = os.environ.get("CUDA_HOME", "/usr/local/cuda") + "/include"


@pytest.fixture(scope="module")
def checker(tmp_path_factory):
    if not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")):
        pytest.skip("CUDA headers not found")
    exe = str(tmp_path_factory.mktemp("hostcheck") / "host_traverse_check")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I" + CUDA_INC, "-I" + os.path.join(ROOT, "include"), "-o", exe,
                           os.path.join(CSRC, "tools", "host_traverse_check.cpp"), os.path.join(CSRC, "bvh.cpp")])
    return exe


def _dump(path, tris, rays):
    tr = np.concatenate([tris[:, 0], tris[:, 1] - tris[:, 0], tris[:, 2] - tris[:, 0]], 1).astype(np.float32)
    with open(path, "wb") as f:
        f.write(np.array([len(tr), len(rays)], np.uint32).tobytes())
        f.write(tr.tobytes())
        f.write(np.ascontiguousarray(rays, np.float32).tobytes())


def _run(exe, path):
    # (opaque modulus, opacity-micromap level): the last two runs give every non-opaque triangle a synthetic micromap (csrc/omm.cuh):
    # OPAQUE micro-triangles must behave like opaque triangles, TRANSPARENT ones like no triangle, in both protocols
    for mod, omm in (("3", "0"), ("-8", "0"), ("3", "3"), ("-8", "2")):
        out = subprocess.run([exe, path, "1000000", mod, omm], capture_output=True, text=True, timeout=600)
        print(out.stdout)
        assert out.returncode == 0, out.stdout + out.stderr
        assert "mismatches: nearest opaque 0, shadow 0, candidates 0" in out.stdout


def test_device_traversal_source_vs_brute_force_soup(checker, tmp_path):
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from gpu_util import random_rays
    rng = np.random.default_rng(3)
    c = (rng.random((4000, 1, 3)) - 0.5) * 2
    tris = c + (rng.random((4000, 3, 3)) - 0.5) * 0.3
    _dump(str(tmp_path / "soup.bin"), tris, random_rays(6000, [-1, -1, -1], [1, 1, 1], seed=11))
    _run(checker, str(tmp_path / "soup.bin"))


def test_device_traversal_source_vs_brute_force_axis_aligned(checker, tmp_path):
    """Flat boxes and grazing rays: a regular grid of axis-aligned quads (zero-thickness nodes, shared edges and vertices),
    rays along the axes, along the planes, through vertices and edges, and starting on the surfaces."""
    g = np.arange(-4, 5, dtype=np.float64) * 0.25
    quads = []
    for k, z in enumerate(g[::2]):                      # layers of z-planes, x-planes and y-planes
        for x0 in g[:-1]:
            for y0 in g[:-1]:
                p = np.array([[x0, y0, z], [x0 + 0.25, y0, z], [x0 + 0.25, y0 + 0.25, z], [x0, y0 + 0.25, z]])
                for perm in ((0, 1, 2), (2, 0, 1), (1, 2, 0))[k % 3:k % 3 + 1]:
                    q = p[:, perm]
                    quads.append([q[0], q[1], q[2]])
                    quads.append([q[0], q[2], q[3]])
    tris = np.array(quads)
    rng = np.random.default_rng(5)
    rays = np.zeros((5000, 8), np.float32)
    o = rng.choice(g, size=(5000, 3)) + rng.choice([0.0, 0.0, 0.125, 1e-6], size=(5000, 3))   # on grid lines, cell centres, just off
    d = rng.choice([-1.0, 0.0, 1.0, 0.5, -0.25], size=(5000, 3))
    d[(d == 0).all(1)] = [0.0, 0.0, 1.0]
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    rays[:, 0:3], rays[:, 4:7], rays[:, 7] = o - 2.0 * d * (rng.random((5000, 1)) > 0.3), d, 1e32
    _dump(str(tmp_path / "grid.bin"), tris, rays)
    _run(checker, str(tmp_path / "grid.bin"))


def test_device_bsdf_source_matches_oracle_bit_for_bit(tmp_path, oracle_mod):
    """csrc/bsdf.cuh (bsdfEvaluate / bsdfSample, FEAT_ALL: diffuse, diffuse transmission, specular, metal, rough and thin-walled
    transmission, clearcoat, sheen, iridescence, anisotropy) compiled for the host with -ffp-contract=off and fed 30 000 random
    records: every output equals the oracle's (oracle/bsdf.h) bit for bit -- both then share one libm, so this pins the two
    SOURCES against each other; on the GPU only CUDA's libm differs (test_bsdf_parity, 2e-4)."""
    if not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")):
        pytest.skip("CUDA headers not found")
    sys.path.insert(0, ROOT)
    from vk_gltf_renderer_b200 import bsdf_io
    exe = str(tmp_path / "host_bsdf_check")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-I" + CUDA_INC, "-o", exe, os.path.join(CSRC, "tools", "host_bsdf_check.cpp")])
    o = oracle_mod.Oracle()
    rec = bsdf_io.random_records(30000, seed=99)
    ev, sm = o.bsdf_eval(rec), o.bsdf_sample(rec)
    simple = o.bsdf_sample_simple(rec)   # the shadow catcher's continuation BSDF: both lobes and the absorbed case occur
    assert {0, 9, 10} <= set(simple[:, 7].astype(int).tolist()) and np.isfinite(simple).all()
    lit = simple[:, 7] != 0
    assert (simple[lit, 6] > 0).all() and (simple[lit, 3:6] >= 0).all() and simple[lit, 3:6].max() < 50.0
    assert len(set(sm[:, 7].astype(int).tolist())) >= 4 and (ev[:, 6] > 0).mean() > 0.2
    path = str(tmp_path / "records.bin")
    with open(path, "wb") as f:
        f.write(np.array([len(rec)], np.uint32).tobytes())
        f.write(rec.tobytes())
        f.write(ev.tobytes())
        f.write(sm.tobytes())
        f.write(simple.tobytes())
    out = subprocess.run([exe, path], capture_output=True, text=True, timeout=600)
    print(out.stdout)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "eval mismatches 0, sample mismatches 0" in out.stdout and "bsdfSampleSimple mismatches 0" in out.stdout


def test_device_refit_source_vs_brute_force(tmp_path):
    """csrc/refit.cuh (re-quantisation of a node from its children's boxes, bottom-up by level) compiled for the host: after a third
    of the triangles moved, the refitted tree -- walked by the device traversal source -- returns the brute-force nearest hit over
    the moved triangles for every ray, bit for bit (tools/host_refit_check.cpp)."""
    if not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")):
        pytest.skip("CUDA headers not found")
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from gpu_util import random_rays
    exe = str(tmp_path / "host_refit_check")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I" + CUDA_INC, "-I" + os.path.join(ROOT, "include"), "-o", exe,
                           os.path.join(CSRC, "tools", "host_refit_check.cpp"), os.path.join(CSRC, "bvh.cpp")])
    rng = np.random.default_rng(3)
    c = (rng.random((3000, 1, 3)) - 0.5) * 2
    tris = c + (rng.random((3000, 3, 3)) - 0.5) * 0.3
    _dump(str(tmp_path / "soup.bin"), tris, random_rays(4000, [-1, -1, -1], [1, 1, 1], seed=11))
    out = subprocess.run([exe, str(tmp_path / "soup.bin")], capture_output=True, text=True, timeout=600)
    print(out.stdout)
    assert out.returncode == 0 and "mismatches after refit: 0" in out.stdout, out.stdout + out.stderr


def test_device_lbvh_build_source_vs_brute_force(tmp_path):
    """csrc/lbvh.cuh (the DEVICE builder: Morton keys, bitonic sort, Karras radix tree, bottom-up fit, level-wise collapse into
    compressed 8-wide nodes) run on the host thread after thread: every triangle of the subset is emitted once and the tree --
    walked by the device traversal source -- returns the brute-force nearest hit for every ray, bit for bit
    (tools/host_lbvh_check.cpp)."""
    if not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")):
        pytest.skip("CUDA headers not found")
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from gpu_util import random_rays
    exe = str(tmp_path / "host_lbvh_check")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I" + CUDA_INC, "-I" + os.path.join(ROOT, "include"), "-o", exe, os.path.join(CSRC, "tools", "host_lbvh_check.cpp")])
    rng = np.random.default_rng(7)
    c = (rng.random((5000, 1, 3)) - 0.5) * 2
    tris = c + (rng.random((5000, 3, 3)) - 0.5) * 0.25
    tris[:40] = tris[0]  # coincident triangles: identical Morton codes, unique keys by index
    _dump(str(tmp_path / "soup.bin"), tris, random_rays(4000, [-1, -1, -1], [1, 1, 1], seed=13))
    out = subprocess.run([exe, str(tmp_path / "soup.bin")], capture_output=True, text=True, timeout=600)
    print(out.stdout)
    assert out.returncode == 0 and "mismatches: 0" in out.stdout, out.stdout + out.stderr
