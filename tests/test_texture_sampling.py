"""The CPU oracle's texture sampler against the float64 Vulkan-sampler restatement in texref.py, over every wrap pair,
the glTF filter combinations, non-power-of-two / thin / single-texel shapes, texel edges, far-away coordinates, gradients on
and off level and rounding boundaries, KHR_texture_transform, TEXCOORD_1 and the "no texture" slot.  The same sweep runs
on the device in test_gpu_textures.py; the lookups go through the production getTexture / sampleLevel0 of each side
(oracle_texture_lookup, b200pt_texture_lookup)."""
import math

import numpy as np
import pytest

import texref as tr
from vk_gltf_renderer_b200 import tex_io

# (w, h); the two large ones get a subset of the sampler states (their chains are big on the CPU side)
SIZES = [(1, 1), (1, 7), (7, 1), (3, 5), (5, 3), (7, 7), (4, 4), (9, 17), (23, 37), (8, 1024), (1024, 8), (64, 64)]
LARGE = [(333, 129), (2048, 2048)]
# (magFilter, minFilter): default, both NEAREST, both LINEAR, every mipmap minFilter, the nearest mip mode that magFilter
# 9728 selects, and magFilter 9986 (NEAREST in getSampler's table)
FILTERS = [(-1, -1), (9728, 9728), (9729, 9729), (9729, 9984), (9729, 9985), (9728, 9986), (9728, 9987), (9729, 9987),
           (9986, 9729)]
WRAP_PAIRS = [(s, t) for s in tr.WRAPS for t in tr.WRAPS]
READBACK = (tr.REPEAT, tr.REPEAT, 9728, 9728)  # nearest level selection + nearest filter: every level reads back texel by texel
ROT30 = (math.cos(math.pi / 6), math.sin(math.pi / 6), -math.sin(math.pi / 6), math.cos(math.pi / 6), 0.3, -0.2)
TRANSFORMS = [(4.0, 0.0, 0.0, 0.25, 0.0, 0.0), ROT30]
EPS = 1e-6           # lambda this close to a level / rounding boundary may land on either side
TOL = 2e-6           # absolute, rgba


class Sweep:
    """One scene holding every (image, sampler) texture of the sweep, one identity texture info per texture, plus
    transformed / TEXCOORD_1 infos on a few textures and a "none" info; `queries` are the lookup records and what the
    reference needs to answer them."""

    def __init__(self, large=True, seed=7):
        from vk_gltf_renderer_b200.scene import Scene
        rng = np.random.default_rng(seed)
        s = Scene()
        s.add_material()
        s.add_primitive([[0, 0, 0], [1, 0, 0], [0, 1, 0]], [[0, 1, 2]], uv0=[[0, 0], [1, 0], [0, 1]])
        s.add_node(0, 0)
        self.scene, self.images, self.textures = s, [], []
        shapes = [(wh, srgb) for wh in SIZES for srgb in (False, True)]
        if large:
            shapes += [(LARGE[0], False), (LARGE[0], True), (LARGE[1], True)]
        for (w, h), srgb in shapes:
            img = rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
            img[0, 0, 3], img[-1, -1, 3] = 0, 255   # alpha spans 0..255
            im = dict(w=w, h=h, srgb=srgb, rgba8=img)
            if w * h <= 64 * 64 * 4:
                states = [(ws, wt, mf, nf) for (ws, wt) in WRAP_PAIRS for (mf, nf) in FILTERS]
            elif w < 1000:
                states = [(ws, wt, -1, -1) for (ws, wt) in WRAP_PAIRS] + [(tr.REPEAT, tr.REPEAT, mf, nf) for (mf, nf) in FILTERS[1:]]
            else:
                states = [READBACK, (tr.CLAMP_TO_EDGE, tr.MIRRORED_REPEAT, 9729, 9987), (tr.MIRRORED_REPEAT, tr.REPEAT, 9728, 9986)]
            im["readback"] = None
            for st in states:
                t = s.add_texture(img, srgb=srgb, wrapS=st[0], wrapT=st[1], magFilter=st[2], minFilter=st[3])
                slot = s.add_texture_info(t, 0)
                self.textures.append(dict(image=len(self.images), tex=t, slot=slot, state=st))
                if st == READBACK:
                    im["readback"] = slot
            assert im["readback"] is not None
            self.images.append(im)
        self.none_slot = s.add_texture_info(-1, 0)
        self.queries = self._queries(rng)

    def _uv(self, w, h, rng):
        n = max(w, h)
        uni = rng.uniform(-4, 5, (48, 2))
        ku = np.array([-w - 1, -1, 0, 1, w // 2, w - 1, w, w + 1, 2 * w], np.float64)
        kv = np.array([-h - 1, -1, 0, 1, h // 2, h - 1, h, h + 1, 2 * h], np.float64)
        eu = np.concatenate([ku / w, (ku + 0.5) / w]).astype(np.float32)
        ev = np.concatenate([kv / h, (kv + 0.5) / h]).astype(np.float32)
        edges = np.stack([rng.choice(eu, 48), rng.choice(ev, 48)], 1)
        sp = np.array([0.0, -0.0, 1.0, np.nextafter(np.float32(0), np.float32(-1)), np.nextafter(np.float32(1), np.float32(0))], np.float32)
        special = np.stack(np.meshgrid(sp, sp), -1).reshape(-1, 2)
        # far away: up to 1e4, and where fp32 still resolves half a texel of the largest level (|u*w| < 2^22)
        far = rng.uniform(-1, 1, (12, 2)) * min(1e4, 2.0 ** 22 / n)
        return np.concatenate([uni, edges, special, far]).astype(np.float32)

    def _queries(self, rng):
        """per texture: mode-1 (level 0) records and mode-0 records with the lambda targets below, then the transformed,
        TEXCOORD_1 and "none" records on a few textures"""
        recs, meta = [], []

        def add(r, k, kind, xf=(1, 0, 0, 1, 0, 0), targeted=None):
            recs.append(r)
            meta.append(dict(tex=k, kind=kind, xf=np.asarray(xf, np.float32), n=len(r),
                             targeted=np.zeros(len(r), bool) if targeted is None else targeted))
        for k, t in enumerate(self.textures):
            im = self.images[t["image"]]
            w, h = im["w"], im["h"]
            uv = self._uv(w, h, rng)
            q = tr.num_levels(w, h) - 1
            # lambda targets: none, magnification, exactly 0, levels, nearest-mip rounding points, fractional, beyond the chain
            lams = [None, -1.3, 0.0, 1.0, 2.0, 0.5, 1.5, 2.5, 0.37, 1.71, q + 2.0] + list(rng.uniform(0, q + 1, 5))
            grad = np.array([0.0 if l is None else np.float32(2.0 ** l / max(w, h)) for l in lams], np.float32)
            pick = np.arange(len(uv)) % len(grad)
            on_purpose = np.array([l is not None and l <= q and l * 2 == round(l * 2) for l in lams])
            add(tex_io.records(t["slot"], uv, mode=tex_io.SAMPLE_LEVEL0, tc1=uv + 0.25), k, "level0")
            add(tex_io.records(t["slot"], uv, tex_grad=grad[pick], tc1=uv + 0.25), k, "grad", targeted=on_purpose[pick])
        # KHR_texture_transform (scale, rotation + offset) and TEXCOORD_1 on a few textures (anisotropic gradients)
        picks = [k for k, t in enumerate(self.textures) if (self.images[t["image"]]["w"], self.images[t["image"]]["h"]) in ((5, 3), (23, 37), (64, 64))
                 and t["state"] in ((tr.MIRRORED_REPEAT, tr.CLAMP_TO_EDGE, 9729, 9987), (tr.CLAMP_TO_EDGE, tr.REPEAT, 9728, 9986))]
        assert len(picks) == 12
        for k in picks:
            t = self.textures[k]
            im = self.images[t["image"]]
            uv = self._uv(im["w"], im["h"], rng)
            g = (np.float32(2.0) ** rng.uniform(-3, math.log2(max(im["w"], im["h"])) + 1, len(uv)).astype(np.float32)) / max(im["w"], im["h"])
            g[::5] = 0
            for xf in TRANSFORMS:
                slot = self.scene.add_texture_info(t["tex"], 0, xf)
                add(tex_io.records(slot, uv, tex_grad=g, tc1=uv * 3), k, "grad", xf)
                add(tex_io.records(slot, uv, mode=tex_io.SAMPLE_LEVEL0, tc1=uv * 3), k, "level0")
            slot = self.scene.add_texture_info(t["tex"], 1)
            add(tex_io.records(slot, uv * 3 - 1, tex_grad=g, tc1=uv), k, "grad")
            add(tex_io.records(slot, uv * 3 - 1, mode=tex_io.SAMPLE_LEVEL0, tc1=uv), k, "level0")
        uv = rng.uniform(-2, 3, (32, 2))
        add(tex_io.records(self.none_slot, uv, tex_grad=0.01), -1, "none")
        add(tex_io.records(self.none_slot, uv, mode=tex_io.SAMPLE_LEVEL0), -1, "none")
        self.meta = meta
        return np.concatenate(recs)


def read_levels(lookup, sweep, im):
    """every stored level of image `im` (uint8 [h, w, 4] each) read back texel by texel through the lookup function,
    plus the level the sampler settles on for a lambda beyond the chain"""
    w, h = im["w"], im["h"]
    n = max(w, h)
    levels = []
    for l in range(tr.num_levels(w, h)):
        lw, lh = tr.level_size(w, h, l)
        ys, xs = np.mgrid[0:lh, 0:lw]
        uv = np.stack([(xs.ravel() + 0.5) / lw, (ys.ravel() + 0.5) / lh], 1)
        rgba = lookup(tex_io.records(im["readback"], uv, tex_grad=0.0 if l == 0 else np.float32(2.0 ** l / n))).reshape(lh, lw, 4)
        u8 = tr.encode_to_u8(rgba, im["srgb"])
        assert np.abs(tr.decode(u8, im["srgb"]) - rgba).max() < 1e-6      # every readback is one stored texel
        levels.append(u8)
    beyond = lookup(tex_io.records(im["readback"], [[0.1, 0.2], [0.7, 0.9], [-3.3, 4.1]], tex_grad=np.float32(2.0 ** (len(levels) + 2) / n)))
    return levels, beyond


def check_chain(levels, beyond, im):
    """level 0 is the image; every further level is the float64 blit of the stored previous one, exact except one 8-bit
    step on a .5 tie; sizes max(1, w >> l); floor(log2(max(w, h))) + 1 levels, a larger lambda stays on the last.
    Returns the number of tie texels."""
    w, h = im["w"], im["h"]
    assert len(levels) == tr.num_levels(w, h)
    assert np.array_equal(levels[0], im["rgba8"])
    ties = 0
    for l in range(1, len(levels)):
        assert levels[l].shape[:2] == tr.level_size(w, h, l)[::-1]
        exact = tr.blit_level(levels[l - 1], im["srgb"])
        diff = levels[l].astype(np.int64) - tr.requantise(exact).astype(np.int64)
        # an even side halves exactly and the blit lands on exact .5 ties; an odd side maps destination centres to
        # positions (x + 1/2) * w / w' that fp32 (and the hardware blit) resolves to about max(w, h) * 2^-23 of a texel
        ph, pw = levels[l - 1].shape[:2]
        window = 1e-4 if pw % 2 == 0 and ph % 2 == 0 or max(pw, ph) == 1 else 1e-4 + 255 * max(pw, ph) * 2.0 ** -23
        on_tie = np.abs(exact - np.floor(exact) - 0.5) < window
        assert np.abs(diff).max() <= 1, (w, h, l)
        assert on_tie[diff != 0].all(), (w, h, l, int((diff != 0).sum()))
        ties += int((diff != 0).sum())
    assert levels[-1].shape[:2] == (1, 1)
    assert np.abs(beyond - tr.decode(levels[-1][0, 0], im["srgb"])).max() < 1e-6
    return ties


def reference(sweep, stored):
    """texref's answer for every query, and per query (float64 lambda, on-a-boundary flag, second admissible answer);
    `stored` maps image -> its stored levels.  A query on a boundary is checked against both sides of it."""
    ref = np.empty((len(sweep.queries), 4))
    sweep.targeted = np.concatenate([m["targeted"] for m in sweep.meta])
    alt = np.empty_like(ref)
    lam = np.full(len(sweep.queries), np.nan)
    edge = np.zeros(len(sweep.queries), bool)
    i = 0
    for m in sweep.meta:
        r = sweep.queries[i:i + m["n"]]
        sl = slice(i, i + m["n"])
        i += m["n"]
        if m["kind"] == "none":
            ref[sl] = alt[sl] = 1.0
            continue
        t = sweep.textures[m["tex"]]
        st = t["state"]
        R = tr.TexRef(stored[t["image"]], sweep.images[t["image"]]["srgb"], *st)
        ti = sweep.scene.texture_infos[int(r[0, 0])]
        tc = np.where(ti.texCoord == 1, r[:, 4:6], r[:, 2:4]).astype(np.float32)
        if m["kind"] == "level0":
            ref[sl] = alt[sl] = R.sample(tc)
            continue
        # getTexture: the uv transform and the gradient footprint in fp32, as the shader forms them
        xf, g = m["xf"], r[:, 6]
        tt = np.stack([xf[0] * tc[:, 0] + xf[2] * tc[:, 1] + xf[4], xf[1] * tc[:, 0] + xf[3] * tc[:, 1] + xf[5]], 1).astype(np.float32)
        ddx, ddy = np.stack([xf[0] * g, xf[1] * g], 1), np.stack([xf[2] * g, xf[3] * g], 1)
        l = np.where(g > 0, R.lod(ddx, ddy), np.nan)
        on = R.lod_boundaries(l, EPS)
        b = np.where(np.abs(l - np.round(l)) < EPS, np.round(l), np.floor(l) + 0.5)
        lo, hi = np.where(on, b - 1e-9, l), np.where(on, b + 1e-9, l)
        nog = ~(g > 0)
        ref[sl] = R.sample(tt, np.where(nog, -1.0, lo))
        alt[sl] = R.sample(tt, np.where(nog, -1.0, hi))
        lam[sl], edge[sl] = l, on
    return ref, alt, lam, edge


def compare(got, ref, alt, lam, edge, tag):
    """within TOL of texref (either side of a boundary for the queries on one); returns the summary counts"""
    assert np.isfinite(got).all()
    err = np.minimum(np.abs(got - ref).max(1), np.abs(got - alt).max(1))
    bad = np.flatnonzero(err > TOL)
    assert len(bad) == 0, (tag, len(bad), bad[:5], err[bad[:5]], lam[bad[:5]])
    mip = np.isfinite(lam) & (lam > 0)
    return dict(queries=len(got), mip=int(mip.sum()), on_boundary=int(edge.sum()), max_err=float(err.max()))


@pytest.fixture(scope="module")
def sweep():
    return Sweep()


@pytest.fixture(scope="module")
def oracle_sweep(sweep, oracle_mod):
    o = oracle_mod.Oracle()
    o.set_scene(sweep.scene)
    stored, ties = {}, 0
    for k, im in enumerate(sweep.images):
        levels, beyond = read_levels(o.texture_lookup, sweep, im)
        ties += check_chain(levels, beyond, im)
        stored[k] = levels
    return o, stored, ties


def test_oracle_mip_chain_matches_the_float64_blit(oracle_sweep):
    _, _, ties = oracle_sweep
    print("oracle mip chain: texels differing from the float64 blit by one step on a .5 tie:", ties)


def test_oracle_sampler_matches_float64_reference(sweep, oracle_sweep):
    o, stored, _ = oracle_sweep
    got = o.texture_lookup(sweep.queries)
    ref, alt, lam, edge = reference(sweep, stored)
    s = compare(got, ref, alt, lam, edge, "oracle")
    print("oracle vs texref:", s)
    assert s["mip"] > 0.3 * s["queries"]
    # the sweep puts lambda on 0, on levels and on k + 1/2 on purpose; among the other gradients boundaries are rare
    other = np.isfinite(lam) & ~sweep.targeted
    print("lambda within %g of a boundary: %d targeted, %d of %d others" % (EPS, (edge & sweep.targeted).sum(), (edge & other).sum(), other.sum()))
    assert (edge & other).sum() <= 1e-3 * other.sum()
    assert (edge & sweep.targeted).sum() > 0
    # the white "none" slot, and a slot outside the scene is refused
    assert (got[sweep.queries[:, 0] == sweep.none_slot] == 1.0).all()
    with pytest.raises(ValueError):
        o.texture_lookup(tex_io.records(len(sweep.scene.texture_infos), [[0.5, 0.5]]))


def test_sampler_mapping_follows_get_sampler():
    """mip mode from magFilter (9728 -> nearest), NEAREST for 9728 / 9984 / 9986 in either slot, LINEAR for the rest
    and for an unset filter"""
    assert tr.sampler_modes(-1, -1) == (True, True, True)
    assert tr.sampler_modes(9728, 9987) == (False, True, False)
    assert tr.sampler_modes(9729, 9984) == (True, False, True)
    assert tr.sampler_modes(9986, 9729) == (False, True, False)
    assert [int(tr.wrap(i, 3, tr.MIRRORED_REPEAT)) for i in range(-4, 8)] == [2, 2, 1, 0, 0, 1, 2, 2, 1, 0, 0, 1]
    assert [int(tr.wrap(i, 3, tr.CLAMP_TO_EDGE)) for i in (-2, 0, 2, 5)] == [0, 0, 2, 2]
    assert [int(tr.wrap(i, 3, tr.REPEAT)) for i in (-4, -1, 0, 3, 4)] == [2, 2, 0, 0, 1]
