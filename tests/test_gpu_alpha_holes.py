"""-m gpu alpha holes (csrc/alpha_caps.cuh): a candidate whose micro-triangle is transparent everywhere passes a closest-hit test only
when its draw is exactly 0.  A walk whose kept candidates are all caps or holes runs the any-hit loop itself, from the seed alone.  Seeds
are chosen so that draw k of every ray is exactly 0 (k = 0 .. 7: in the main walk, in a continuation round and in the in-kernel fallback),
so that holes are accepted; a handle with caps and holes must answer exactly what a handle without them (B200PT_ALPHA_CAPS=0) answers,
hits, seeds and transmission bit for bit."""
import numpy as np
import pytest

from test_gpu_alpha_caps import _deep_layers, _draws, _handle, _rays
from test_gpu_scene_edits import _clone

pytestmark = pytest.mark.gpu

A, C, M = 747796405, 2891336453, 1 << 32


def _zero_states():
    """the 512 pcg states (vec.cuh) right after a step whose rnd() is exactly 0 (output >> 9 == 0), by inverting the output permutation"""
    r = np.arange(512, dtype=np.uint64)
    w = r ^ (r >> 22)
    g = (w * pow(277803737, -1, M)) % M
    sh = (g >> 28) + 4
    prev = g.copy()
    for _ in range(8):
        prev = g ^ (prev >> sh)
    return prev


def _pcg_out(state):
    prev = (state.astype(np.uint64) * A + C) % M
    word = (((prev >> ((prev >> 28) + 4)) ^ prev) * 277803737) % M
    return prev, (word >> 22) ^ word


def _seeds_zero_at(k, n):
    """seeds whose draw k (0-based) is exactly 0"""
    s = _zero_states()[np.arange(n) % 512]
    inv = pow(A, -1, M)
    for _ in range(k + 1):
        s = ((s + M - C) * inv) % M
    return s.astype(np.uint32)


def test_zero_draw_states():
    s = _seeds_zero_at(0, 512)
    _, out = _pcg_out(s)
    assert ((out >> 9) == 0).all()


@pytest.mark.parametrize("rounds", [1, 2])
def test_zero_draws_on_holes_change_no_result(std_env, monkeypatch, rounds):
    monkeypatch.setenv("B200PT_CONT_ROUNDS", str(rounds))
    scn, rays, _, tmax = _deep_layers()
    handles = [_handle(_clone(scn), std_env, caps, monkeypatch)[0] for caps in (True, False)]
    accepted_at_k = 0
    for k in range(8):
        seeds = _seeds_zero_at(k, len(rays))
        got, ref = (_rays(pt, rays, seeds, tmax) for pt in handles)
        for key in ("hits", "trans", "seeds"):
            np.testing.assert_array_equal(got[key].view(np.uint32), ref[key].view(np.uint32), err_msg=f"{key} k={k}")
        # rays that drew exactly k + 1 times stopped at the zero draw: their hit is the layer it was drawn for
        d = _draws(seeds, got["seeds"][0])
        accepted_at_k += int((d == k + 1).sum())
    for pt in handles:
        pt.onDetach()
    assert accepted_at_k > 1000, accepted_at_k
