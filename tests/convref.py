"""Float64 restatement of the per-pixel convergence rule (include/b200pt.h b200pt_set_convergence, csrc/converge.cuh) and the
synthetic frame streams the host check of tests/test_convergence.py feeds it.

The device keeps M2 with West's weighted Welford update in fp32.  Here M2 is restated TWO-PASS in float64 from the frames' luminances:
after F frames with weights n_f and luminances c_f, m = sum n_f c_f / N and M2 = sum n_f (c_f - m)^2, which the update equals in exact
arithmetic.  `m2_bound` is a first-order bound on the fp32 recurrence's distance from it."""
import numpy as np

U = 2.0 ** -24  # unit roundoff of fp32


def lum(c):
    return (c[..., 0] + c[..., 1] + c[..., 2]) / 3.0


def frame_means(sums, ns):
    """the frames' clamped sample means c_f = pixSum / numSamples in float64: [F, P, 4]"""
    return np.asarray(sums, np.float64) / np.asarray(ns, np.float64)[:, None, None]


def two_pass(c_lum, ns, frames):
    """(m, M2) of every pixel after its first `frames` frames, two-pass in float64; c_lum [F, P]"""
    w = np.asarray(ns[:frames], np.float64)[:, None]
    x = c_lum[:frames]
    m = (w * x).sum(0) / w.sum()
    return m, (w * (x - m) ** 2).sum(0)


def rel_error(m2, frames, samples, m, floor):
    """e = sqrt(M2 / ((F - 1) N)) / max(m, floor), +inf while F < 2"""
    if frames < 2:
        return np.full(np.shape(m2), np.inf)
    return np.sqrt(np.maximum(m2, 0.0) / ((frames - 1) * samples)) / np.maximum(m, floor)


def m2_bound(c_lum, ns):
    """per frame f (after it) and pixel: a first-order bound on |M2_fp32 - M2| for the fp32 recurrence.
    The fp32 running mean's luminance is off by at most eps_m(f) = 4u f max|c| + 2u |m| (one fold per frame, four roundings each,
    plus the luminance's two), a frame mean's by eps_c = 3u |c|; each update term n (c - m_prev)(c - m) then errs by at most
    n [(|a| + eps_c + eps_m(f-1))(|b| + eps_c + eps_m(f))(1 + 3u) - |a||b|], and the running sum by u |M2| per frame."""
    c_lum = np.asarray(c_lum, np.float64)
    F = c_lum.shape[0]
    w = np.asarray(ns, np.float64)[:, None]
    N = np.cumsum(w[:, 0])[:, None]
    m = np.cumsum(w * c_lum, axis=0) / N             # exact running mean after each frame
    cmax = np.maximum.accumulate(np.abs(c_lum), axis=0)
    eps_m = 4 * U * np.arange(1, F + 1)[:, None] * cmax + 2 * U * np.abs(m)
    eps_c = 3 * U * np.abs(c_lum)
    bound = np.zeros_like(c_lum)
    m2 = np.zeros(c_lum.shape[1])
    acc = np.zeros(c_lum.shape[1])
    for f in range(1, F):
        a, b = np.abs(c_lum[f] - m[f - 1]), np.abs(c_lum[f] - m[f])
        term = w[f] * ((a + eps_c[f] + eps_m[f - 1]) * (b + eps_c[f] + eps_m[f]) * (1 + 3 * U) - a * b)
        m2 += w[f] * (c_lum[f] - m[f - 1]) * (c_lum[f] - m[f])
        acc += term + U * np.abs(m2)
        bound[f] = acc
    return bound


# ---- synthetic streams ----------------------------------------------------------------------------------------------------------
def pixel_kinds(rng, per_kind):
    """per pixel: (mean RGB, relative noise, heavy tail) for the kinds the rule must handle"""
    kinds = []
    for _ in range(per_kind):
        kinds.append((rng.uniform(0.05, 2.0, 3), rng.uniform(0.05, 3.0), False))   # ordinary noisy pixels
        kinds.append((rng.uniform(0.05, 2.0, 3), 0.0, False))                      # zero variance
        kinds.append((np.zeros(3), 0.0, False))                                    # black
        kinds.append((rng.uniform(1e-6, 1e-4, 3), rng.uniform(0.1, 2.0), False))   # dim, below the floor
        kinds.append((rng.uniform(0.2, 1.0, 3), 1.0, True))                        # rare samples at the firefly clamp
        kinds.append((rng.uniform(0.9e4, 1.1e4, 3), rng.uniform(0.001, 0.2), False))  # near 1e4
    return kinds


def stream(rng, kinds, ns, clamp=10.0):
    """pixel sums [F, P, 4] (float32, summed sample by sample like P.pixSum) for the given numSamples per frame; the heavy-tailed
    kind's rare samples sit exactly at the firefly clamp's luminance"""
    P = len(kinds)
    mean = np.array([k[0] for k in kinds], np.float64)
    noise = np.array([k[1] for k in kinds], np.float64)
    heavy = np.array([k[2] for k in kinds])
    out = np.zeros((len(ns), P, 4), np.float32)
    for f, n in enumerate(ns):
        s = np.zeros((P, 4), np.float32)
        for _ in range(n):
            g = rng.standard_normal((P, 1))
            v = np.maximum(mean * (1.0 + noise[:, None] * g), 0.0)
            spike = heavy[:, None] & (rng.random((P, 1)) < 0.02)
            v = np.where(spike, mean * (clamp / np.maximum(mean.sum(1, keepdims=True) / 3.0, 1e-30)), v)
            r = np.concatenate([v, np.ones((P, 1))], 1).astype(np.float32)
            s = (s + r).astype(np.float32)
        out[f] = s
    return out
