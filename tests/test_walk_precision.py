"""Tree walks against brute force where their rounding matters (-m "not gpu"): nodes far from the ray origin relative to their
size, flat nodes, slivers, coincident triangles, +-0 and clamped direction components, origins on a surface, segments ending at
their hit (tests/walkcases.py).

The device walk source (csrc/traverse.cuh, compiled for the host by tools/host_traverse_check.cpp) must return exactly what the
brute force with the kernel's own triangle test returns: the nearest opaque hit, the candidates in (t, id) order across
continuation walks, and the shadow protocol, on the host builder's tree, the device builder's tree and a refitted tree, without
and with opacity micromaps.  The brute force itself is pinned by a float64 classification of every (ray, triangle) pair, and the
CPU oracle's walk must find every brute-force hit too.

The node test is conservative for triangle tests whose t errs by less than RHO_MAX e D along the ray (traverse.cuh, kWalkEps;
e = 2^-24, D the L1 distance from the origin to v0).  Hits seen nearly edge-on and hits on slivers exceed that: there the fp32 t
itself is off by up to a few 1e-3 of t (sin(phi) cos(theta) below ~1e-4), more than any node widening that keeps far nodes tight
could cover.  The rays that meet such a hit are held to the brute force separately, with a bound on their share and on their
mismatches."""
import functools
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "vk_gltf_renderer_b200", "csrc")
CUDA_INC = os.environ.get("CUDA_HOME", "/usr/local/cuda") + "/include"
sys.path.insert(0, os.path.join(ROOT, "tests"))
import walkcases as W  # noqa: E402

# t error of the triangle test, in units of e |org - v0|_1 / |dir|, that the node test's widening covers: 256 - 8 (slab
# arithmetic, traverse.cuh) less the origin-shift part of the triangle test, rounded down
RHO_MAX = 192.0
TREES = {0: "host builder", 1: "device builder", 2: "refitted"}
PROTOCOLS = (("-8", "0"), ("3", "2"))  # (opaque modulus, micromap level): 7/8 non-opaque without micromaps, 1/3 with level 2


def compile_checker(out_dir):
    exe = os.path.join(str(out_dir), "host_traverse_check")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I" + CUDA_INC, "-I" + os.path.join(ROOT, "include"), "-o", exe,
                           os.path.join(CSRC, "tools", "host_traverse_check.cpp"), os.path.join(CSRC, "bvh.cpp")])
    return exe


def run_checker(exe, path, mod="-8", omm="0", tree=0, hits=None):
    """(nearest opaque, shadow, candidates) mismatch counts of one run on every ray's own (tmin, tmax)"""
    args = [exe, path, "100000000", mod, omm, str(tree), "1"] + ([hits] if hits else [])
    out = subprocess.run(args, capture_output=True, text=True, timeout=900)
    assert out.returncode in (0, 1) and "mismatches:" in out.stdout, out.stdout + out.stderr
    line = out.stdout.strip().splitlines()[-1]
    assert "deepest stack" in line and "of 28" in line and " 28 of" not in line, line
    tail = line.split("mismatches:")[1]
    return tuple(int(x.split()[-1]) for x in tail.split(","))


@pytest.fixture(scope="module")
def checker(tmp_path_factory):
    if not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")):
        pytest.skip("CUDA headers not found")
    return compile_checker(tmp_path_factory.mktemp("walkcheck"))


class Cases:
    """per family: the dump, the brute-force hits and the split of the rays into well- and ill-conditioned ones"""

    def __init__(self, exe, d):
        self.exe, self.d = exe, d

    @functools.lru_cache(maxsize=None)
    def get(self, name):
        return brute_force(self.exe, self.d, name, *W.case(name))


def brute_force(exe, d, tag, v, R):
    """the kernel-arithmetic brute force of (v, R): every hit, its t error, the rays with an ill-conditioned hit, the nearest hit
    (t, id) of every ray (inf, -1 on a miss), and dumps of the well- and ill-conditioned rays"""
    path = os.path.join(d, tag + ".bin")
    W.dump(path, v, R)
    hits = os.path.join(d, tag + ".hits")
    run_checker(exe, path, "-1", "0", 0, hits)
    ids, fl = W.read_hits(hits)
    rho = t_error(W.records(v), R, ids, fl[:, 0])
    ill = np.unique(ids[rho > RHO_MAX, 0])
    well = np.setdiff1d(np.arange(len(R)), ill)
    paths = {}
    for part, rows in (("well", well), ("ill", ill)):
        paths[part] = os.path.join(d, "%s_%s.bin" % (tag, part))
        W.dump(paths[part], v, R[rows])
    near_t = np.full(len(R), np.inf, np.float32)
    near_id = np.full(len(R), -1, np.int64)
    order = np.lexsort((ids[:, 1], fl[:, 0]))[::-1]  # the last write per ray is its (t, id)-smallest hit
    near_t[ids[order, 0]] = fl[order, 0]
    near_id[ids[order, 0]] = ids[order, 1]
    return dict(v=v, R=R, ids=ids, fl=fl, rho=rho, ill=ill, well=well, paths=paths, near_t=near_t, near_id=near_id)


@pytest.fixture(scope="module")
def cases(checker, tmp_path_factory):
    return Cases(checker, str(tmp_path_factory.mktemp("walkcases")))


def t_error(rec, R, ids, t32):
    """|t32 - t| |dir| / (e |org - v0|_1) of every brute-force hit, t the float64 intersection of the fp32 ray with the stored plane"""
    rec = rec.astype(np.float64)
    o, d = R[ids[:, 0], 0:3].astype(np.float64), R[ids[:, 0], 4:7].astype(np.float64)
    v0, e1, e2 = rec[ids[:, 1], 0:3], rec[ids[:, 1], 3:6], rec[ids[:, 1], 6:9]
    n = np.cross(e1, e2)
    t = ((v0 - o) * n).sum(1) / (d * n).sum(1)
    return np.abs(t32 - t) * np.linalg.norm(d, axis=1) / (W.EPS * np.abs(o - v0).sum(1))


@pytest.mark.parametrize("name", W.FAMILIES)
def test_float64_classification_pins_the_brute_force(cases, name):
    """Every pair the float64 classification calls a certain hit is a hit of the kernel-arithmetic brute force, and every hit of
    the brute force is a certain or borderline pair (none is a certain miss).  Borderline pairs, mostly the rays aimed at edges
    and vertices, stay rare, and so do the rays with a hit whose t errs by more than the node test's widening covers."""
    c = cases.get(name)
    sure, border, n = W.classify(W.records(c["v"]), c["R"])
    key = lambda a: a[:, 0] * 1_000_003 + a[:, 1]  # noqa: E731
    got = key(c["ids"])
    assert np.isin(key(sure), got).all(), "certain hits the fp32 test missed: %d" % (~np.isin(key(sure), got)).sum()
    allowed = np.union1d(key(sure), key(border))
    assert np.isin(got, allowed).all(), "fp32 hits on certain misses: %d" % (~np.isin(got, allowed)).sum()
    share = len(border) / n
    print("%s: %d pairs, %d certain hits, %d borderline (%.2e), brute-force hits %d, t error max %.1f e D, ill-conditioned rays %d"
          % (name, n, len(sure), len(border), share, len(got), c["rho"].max(), len(c["ill"])))
    # every hit on a sliver is ill-conditioned in u, v and t; the tiles share every edge and vertex a ray is aimed at
    bound = {"slivers": 1e-2, "layers": 5e-3}.get(name, 1e-3)
    assert len(sure) > 0.75 * len(got) and share < bound
    assert len(c["ill"]) <= (0.2 if name == "slivers" else 0.005) * len(c["R"])


@pytest.mark.parametrize("mod,omm", PROTOCOLS)
@pytest.mark.parametrize("tree", sorted(TREES))
@pytest.mark.parametrize("name", W.FAMILIES)
def test_walks_match_brute_force(checker, cases, name, tree, mod, omm):
    """closest protocol with every candidate rejected and shadow protocol, bit for bit, on every ray whose hits the node test's
    widening covers; the few rays beyond it (edge-on hits, slivers) are reported and bounded"""
    c = cases.get(name)
    bad = run_checker(checker, c["paths"]["well"], mod, omm, tree)
    print("%s, %s tree, modulus %s, micromap level %s: mismatches %s on %d rays" % (name, TREES[tree], mod, omm, bad, len(c["R"]) - len(c["ill"])))
    assert bad == (0, 0, 0)
    if len(c["ill"]):
        bad = run_checker(checker, c["paths"]["ill"], mod, omm, tree)
        print("  rays with an ill-conditioned hit: mismatches %s on %d rays" % (bad, len(c["ill"])))
        assert sum(bad) <= max(2, 0.25 * len(c["ill"]))


@pytest.mark.parametrize("name", W.FAMILIES)
def test_oracle_finds_every_brute_force_hit(cases, oracle_mod, name):
    """The CPU oracle's walk on the family as an all-opaque, double-sided scene (synth.triangle_soup): its nearest hit is the
    brute force's nearest (t, id) bit for bit, and its shadow rays are occluded exactly when the segment has a brute-force hit."""
    from vk_gltf_renderer_b200 import synth
    c = cases.get(name)
    scn = synth.triangle_soup(0, vertices=c["v"], double_sided=1)
    o = oracle_mod.Oracle()
    o.set_scene(scn)
    R, want_t, want_id = c["R"], c["near_t"], c["near_id"]
    keep = ~np.isin(np.arange(len(R)), c["ill"])
    hits = o.trace_closest(R)
    got_id = hits.view(np.int32)[:, 3].astype(np.int64)
    miss_c = keep & ((got_id != want_id) | ((want_id >= 0) & (hits[:, 0].view(np.uint32) != want_t.view(np.uint32))))
    tr = o.trace_shadow(R)
    miss_s = keep & ((tr[:, 0] == 0) != (want_id >= 0))
    print("%s: oracle closest mismatches %d, shadow %d of %d rays" % (name, miss_c.sum(), miss_s.sum(), keep.sum()))
    assert miss_c.sum() == 0 and miss_s.sum() == 0
