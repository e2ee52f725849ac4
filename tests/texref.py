"""Float64 restatement of the texel filtering the renderer's sampler implements, for the texture tests.

Written from the Vulkan specification's texel-filtering equations ("Texel Filtering", "Wrapping Operation", "LOD
Operation", "Image Level(s) Selection") and the reference's glTF -> VkSampler mapping (getSampler,
src/gltf_scene_vk.cpp:909-947), not from either implementation:

  * wrap: REPEAT (i mod n), CLAMP_TO_EDGE (clamp to [0, n-1]) and MIRRORED_REPEAT ((n-1) - mirror((i mod 2n) - n));
  * NEAREST picks floor(u*w); LINEAR blends the four texels around u*w - 0.5 with weights frac(u*w - 0.5);
  * lambda = log2(max(|ddx * size|, |ddy * size|)); lambda <= 0 is magnification (level 0, magFilter);
    otherwise it is clamped to the last level, and the mip mode picks level ceil(lambda + 0.5) - 1 (NEAREST) or blends
    floor(lambda) and the next level by frac(lambda) (LINEAR), each sampled with minFilter;
  * sRGB texels decode to linear before filtering (alpha is linear);
  * glTF 9728 / 9984 / 9986 are NEAREST, 9729 / 9985 / 9987 and -1 (unset) LINEAR; the mip mode comes from magFilter.

Two measured rules keep the comparison exact.  The texel-space coordinate is formed in fp32, as the shaders form it: the
product u*w (and v*h) -- in float64 a point exactly on a texel edge lands on the other side -- and, for LINEAR, the
half-texel shift u*w - 1/2, which rounds where it crosses into the next binade (about 1e-5 of a texel at |u*w| ~ 256).
Everything after that is float64.  The mip chain is not rebuilt here: the tests read each level back from the
implementation and check it against `blit_level` applied to the previous level as stored (2x linear blit at the
destination texel centres, clamped, then requantised to 8 bit).  The blit produces exact .5 ties, which the reference's
hardware blit rounds its own way, so a stored texel may differ by one step exactly where `blit_level` lands on a tie.
"""
import numpy as np

REPEAT, CLAMP_TO_EDGE, MIRRORED_REPEAT = 10497, 33071, 33648
WRAPS = (REPEAT, CLAMP_TO_EDGE, MIRRORED_REPEAT)
_LINEAR_FILTER = {-1: True, 9728: False, 9729: True, 9984: False, 9985: True, 9986: False, 9987: True}


def sampler_modes(mag_filter, min_filter):
    """(magnification linear, minification linear, mip mode linear) of a glTF sampler as getSampler builds it"""
    mag = _LINEAR_FILTER[mag_filter]
    return mag, _LINEAR_FILTER[min_filter], mag


def srgb_decode(c):
    c = np.asarray(c, np.float64)
    return np.where(c <= 0.04045, c / 12.92, ((c + 0.055) / 1.055) ** 2.4)


def srgb_encode(c):
    c = np.asarray(c, np.float64)
    return np.where(c <= 0.0031308, c * 12.92, 1.055 * np.maximum(c, 0.0) ** (1.0 / 2.4) - 0.055)


def decode(rgba8, srgb):
    """8-bit texels -> linear float64 [..., 4]"""
    v = np.asarray(rgba8, np.float64) / 255.0
    if srgb:
        v = v.copy()
        v[..., :3] = srgb_decode(v[..., :3])
    return v


def encode_to_u8(lin, srgb):
    """inverse of decode for values that came out of a level-0 or nearest fetch: the nearest 8-bit code per channel"""
    lin = np.asarray(lin, np.float64)
    table = decode(np.repeat(np.arange(256)[:, None], 4, 1), srgb)   # increasing per channel
    out = np.empty(lin.shape, np.uint8)
    for c in range(4):
        mid = (table[1:, c] + table[:-1, c]) / 2
        out[..., c] = np.searchsorted(mid, lin[..., c])
    return out


def wrap(i, n, mode):
    i = np.asarray(i, np.int64)
    if mode == CLAMP_TO_EDGE:
        return np.clip(i, 0, n - 1)
    if mode == MIRRORED_REPEAT:
        a = np.mod(i, 2 * n) - n
        return (n - 1) - np.where(a >= 0, a, -(1 + a))
    assert mode == REPEAT, mode
    return np.mod(i, n)


def level_size(w, h, level):
    return max(1, w >> level), max(1, h >> level)


def num_levels(w, h):
    return int(np.floor(np.log2(max(w, h)))) + 1


def blit_level(prev_u8, srgb):
    """The next level of a stored level (uint8 [h, w, 4]) before requantisation, in 8-bit units (float64 [h', w', 4]):
    vkCmdBlitImage with VK_FILTER_LINEAR, destination texel centres mapped into the source, CLAMP_TO_EDGE, filtered in
    linear space and sRGB-encoded again for sRGB images."""
    h, w = prev_u8.shape[:2]
    nw, nh = max(1, w // 2), max(1, h // 2)
    lin = decode(prev_u8, srgb)
    sx = (np.arange(nw) + 0.5) * (w / nw) - 0.5
    sy = (np.arange(nh) + 0.5) * (h / nh) - 0.5
    x0, y0 = np.floor(sx).astype(np.int64), np.floor(sy).astype(np.int64)
    fx, fy = (sx - x0)[None, :, None], (sy - y0)[:, None, None]
    xa, xb = np.clip(x0, 0, w - 1), np.clip(x0 + 1, 0, w - 1)
    ya, yb = np.clip(y0, 0, h - 1), np.clip(y0 + 1, 0, h - 1)
    top = lin[ya][:, xa] * (1 - fx) + lin[ya][:, xb] * fx
    bot = lin[yb][:, xa] * (1 - fx) + lin[yb][:, xb] * fx
    v = top * (1 - fy) + bot * fy
    if srgb:
        v[..., :3] = srgb_encode(v[..., :3])
    return v * 255.0


def requantise(v255):
    return np.clip(np.floor(v255 + 0.5), 0, 255).astype(np.uint8)


class TexRef:
    """One texture: its stored levels (uint8 [h, w, 4] each, level 0 first) and glTF sampler state."""

    def __init__(self, levels, srgb, wrap_s=REPEAT, wrap_t=REPEAT, mag_filter=-1, min_filter=-1):
        self.levels = [decode(l, srgb) for l in levels]
        self.h0, self.w0 = levels[0].shape[:2]
        self.wrap_s, self.wrap_t = wrap_s, wrap_t
        self.mag_linear, self.min_linear, self.mip_linear = sampler_modes(mag_filter, min_filter)

    @property
    def max_level(self):
        return len(self.levels) - 1

    def sample_level(self, level, uv, linear):
        """uv float32 [n, 2] -> rgba float64 [n, 4] of one level"""
        L = self.levels[level]
        h, w = L.shape[:2]
        uv = np.asarray(uv, np.float32)
        x = (uv[:, 0] * np.float32(w)).astype(np.float64)   # the fp32 texel-space products
        y = (uv[:, 1] * np.float32(h)).astype(np.float64)
        if not linear:
            return L[wrap(np.floor(y), h, self.wrap_t), wrap(np.floor(x), w, self.wrap_s)]
        # the half-texel shift in fp32 too: it rounds where u*w - 1/2 crosses into the next binade
        x = (x.astype(np.float32) - np.float32(0.5)).astype(np.float64)
        y = (y.astype(np.float32) - np.float32(0.5)).astype(np.float64)
        i0, j0 = np.floor(x), np.floor(y)
        a, b = (x - i0)[:, None], (y - j0)[:, None]
        i0, j0 = i0.astype(np.int64), j0.astype(np.int64)
        xs0, xs1 = wrap(i0, w, self.wrap_s), wrap(i0 + 1, w, self.wrap_s)
        ys0, ys1 = wrap(j0, h, self.wrap_t), wrap(j0 + 1, h, self.wrap_t)
        return ((1 - a) * (1 - b) * L[ys0, xs0] + a * (1 - b) * L[ys0, xs1]
                + (1 - a) * b * L[ys1, xs0] + a * b * L[ys1, xs1])

    def lod(self, ddx, ddy):
        """float64 lambda of the (fp32) gradients, [n]"""
        ddx, ddy = np.asarray(ddx, np.float64), np.asarray(ddy, np.float64)
        s = np.array([self.w0, self.h0], np.float64)
        rho = np.maximum(np.linalg.norm(ddx * s, axis=1), np.linalg.norm(ddy * s, axis=1))
        with np.errstate(divide="ignore"):
            return np.log2(rho)

    def sample(self, uv, lam=None):
        """rgba float64 [n, 4]; lam None (no gradient) or float64 lambda per query (from `lod`, or a chosen value)"""
        uv = np.asarray(uv, np.float32).reshape(-1, 2)
        out = self.sample_level(0, uv, self.mag_linear)
        if lam is None:
            return out
        lam = np.broadcast_to(np.asarray(lam, np.float64), (len(uv),))
        minify = lam > 0
        lamc = np.minimum(lam, self.max_level)
        q = self.max_level
        if not self.mip_linear:
            lvl = np.clip(np.ceil(lamc + 0.5) - 1, 0, q).astype(np.int64)
            for l in np.unique(lvl[minify]):
                m = minify & (lvl == l)
                out[m] = self.sample_level(l, uv[m], self.min_linear)
            return out
        l0 = np.floor(lamc).astype(np.int64)
        f = (lamc - l0)[:, None]
        for l in np.unique(l0[minify]):
            m = minify & (l0 == l)
            a = self.sample_level(l, uv[m], self.min_linear)
            l1 = min(l + 1, q)
            b = self.sample_level(l1, uv[m], self.min_linear) if l1 != l else a
            out[m] = a * (1 - f[m]) + b * f[m]
        return out

    def lod_boundaries(self, lam, eps=1e-6):
        """queries whose lambda is within eps of a value where the selection changes: magnification / minification
        (0), a level (integer), a nearest-mip rounding point (k + 1/2) -- where a one-ulp difference in log2 may pick
        the other side"""
        lam = np.asarray(lam, np.float64)
        near_int = np.abs(lam - np.round(lam)) < eps
        near_half = np.abs(lam - (np.floor(lam) + 0.5)) < eps
        return np.isfinite(lam) & (lam > -eps) & (lam < self.max_level + eps) & (near_int | near_half)
