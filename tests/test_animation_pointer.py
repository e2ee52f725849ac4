"""KHR_animation_pointer on the host (animation.sample_pointers / apply_pointers; the reference's AnimationPointerSystem,
src/gltf_animation_pointer.cpp, fed by AnimationSystem::updateAnimation, src/gltf_scene_animation.cpp:377-380).

A hand-written asset animates a base colour, a roughness, an alpha cutoff, an emissive colour, a texture transform's offset, two
material-extension factors, a spot light, a camera and a parent node's visibility, next to channels that must change nothing: a
CUBICSPLINE scalar, a pointer to a node's translation, and malformed pointers.  At times before, on, between and after the keys
and on a zero-length segment:

(a) every sampled value matches `_ref_value`, a float64 restatement of processAnimationChannel / calculateInterpolationFactor
    and the LINEAR / STEP / CUBICSPLINE pointer handlers.  Bound: the implementation evaluates in fp32.  The factor t carries at
    most 3 roundings (time - t0, t1 - t0, the quotient), so |dt| <= 3 eps t.  glm::mix rounds 1 - t, two products and a sum:
    |err| <= |y - x| 3 eps + 4 eps (|x| + |y|) <= 8 eps (|x| + |y|).  The Hermite weights are cubic in t with coefficients up to
    3 and carry about 6 roundings each, times key_delta for the tangent weights; each of the four products and three sums adds one
    more: |err| <= 32 eps (|v0| + |v1| + key_delta (|a| + |b|)).  STEP is exact.
(b) the description apply_pointers makes (materials, texture infos, lights, render-node visibility) is byte-equal to what
    load_gltf makes of the same asset with those values written into its JSON by hand: a texture-info extension replaced, a
    material extension merged, a node's visibility extension replaced, and nothing else;
(c) the oracle's image of the animated scene equals the oracle's image of that static asset, bit for bit.
"""
import base64
import copy
import io
import json

import numpy as np
import pytest

EPS = float(np.finfo(np.float32).eps)
TIMES = (-0.5, 0.0, 0.37, 1.0, 1.6, 2.0, 2.5)    # before, on a key, between, on a key, between, on the last key / zero-length, after
K3 = [0.0, 1.0, 2.0]
K4 = [0.0, 1.0, 2.0, 2.0]                        # a zero-length last segment: at t = 2 the factor is 0, the value key 2's
LIGHT = "/extensions/KHR_lights_punctual/lights/0/"

# (pointer, interpolation, accessor type, key times, outputs); CUBICSPLINE outputs are (in-tangent, value, out-tangent) per key
CHANNELS = [
    ("/materials/0/pbrMetallicRoughness/baseColorFactor", "LINEAR", "VEC4", K3,
     [[0.8, 0.7, 0.6, 1.0], [0.1, 0.9, 0.3, 1.0], [0.95, 0.2, 0.55, 0.9]]),
    ("/materials/0/pbrMetallicRoughness/roughnessFactor", "LINEAR", "SCALAR", K4, [0.6, 0.15, 0.85, 0.05]),
    ("/materials/1/alphaCutoff", "STEP", "SCALAR", K3, [0.3, 0.65, 0.45]),
    ("/materials/0/emissiveFactor", "CUBICSPLINE", "VEC3", K3,
     [[0, 0, 0], [0.1, 0.0, 0.0], [0.5, 0.2, 0.0], [0.3, -0.2, 0.1], [0.6, 0.3, 0.2], [0.1, 0.4, -0.3],
      [-0.2, 0.1, 0.0], [0.2, 0.5, 0.4], [0, 0, 0]]),
    ("/materials/0/pbrMetallicRoughness/metallicFactor", "CUBICSPLINE", "SCALAR", K3,       # no float branch: changes nothing
     [0.0, 0.1, 0.4, 0.2, 0.9, 0.1, 0.3, 0.5, 0.0]),
    ("/materials/1/pbrMetallicRoughness/baseColorTexture/extensions/KHR_texture_transform/offset", "LINEAR", "VEC2", K3,
     [[0.1, 0.2], [0.35, -0.15], [0.0, 0.6]]),
    ("/materials/0/extensions/KHR_materials_emissive_strength/emissiveStrength", "LINEAR", "SCALAR", K3, [2.0, 5.0, 1.5]),
    ("/materials/2/extensions/KHR_materials_transmission/transmissionFactor", "STEP", "SCALAR", K3, [0.0, 0.5, 0.5]),
    (LIGHT + "color", "LINEAR", "VEC3", K3, [[1.0, 0.9, 0.8], [0.2, 1.0, 0.4], [0.9, 0.3, 1.0]]),
    (LIGHT + "intensity", "LINEAR", "SCALAR", K3, [5.0, 8.0, 3.0]),
    (LIGHT + "range", "LINEAR", "SCALAR", K3, [10.0, 6.0, 12.0]),
    (LIGHT + "spot/innerConeAngle", "LINEAR", "SCALAR", K3, [0.2, 0.1, 0.3]),
    (LIGHT + "spot/outerConeAngle", "LINEAR", "SCALAR", K3, [0.6, 0.7, 0.5]),
    ("/cameras/0/perspective/yfov", "LINEAR", "SCALAR", K3, [0.8, 0.5, 1.1]),
    ("/nodes/5/extensions/KHR_node_visibility/visible", "STEP", "SCALAR", [0.0, 1.5, 2.0], [0.0, 0.25, 1.0]),   # shown at 1.5
    ("/nodes/6/translation", "LINEAR", "VEC3", K3, [[0, -0.9, 0.2], [1, 1, 1], [2, 2, 2]]),  # syncNode merges extensions only
    (None, "LINEAR", "SCALAR", K3, [0.0, 1.0, 0.5]),                                        # no KHR_animation_pointer extension
    ("/materials/9/pbrMetallicRoughness/roughnessFactor", "LINEAR", "SCALAR", K3, [0.0, 1.0, 0.5]),   # index out of range
    ("/materials/01x/pbrMetallicRoughness/roughnessFactor", "LINEAR", "SCALAR", K3, [0.0, 1.0, 0.5]),  # index does not parse
    ("/foo/0/roughnessFactor", "LINEAR", "SCALAR", K3, [0.0, 1.0, 0.5]),                      # unknown prefix
]
MOVER, PARENT, CHILD = 7, 5, 6


def _png_data_uri():
    from PIL import Image
    a = np.zeros((8, 8, 4), np.uint8)
    a[..., 0], a[..., 1], a[..., 2] = 200, 120, 60
    a[..., 3] = np.where((np.arange(8)[:, None] // 2 + np.arange(8)[None, :] // 2) % 2 == 0, 255, 110)
    buf = io.BytesIO()
    Image.fromarray(a, "RGBA").save(buf, "PNG")
    return "data:image/png;base64," + base64.b64encode(buf.getvalue()).decode()


def asset_doc():
    """glTF JSON of the test asset: a back wall (material 0), a MASK quad with a transformed texture (material 1), a glass quad whose
    transmission steps 0 -> 0.5 (material 2), a spot light, a camera, a hidden-then-shown parent of a quad, and a morphed quad (node
    7, `mover`) that a translation channel and a weights channel move (the feed of sample_animation)."""
    chunks, views, accessors = [], [], []

    def add(arr, ctype, atype):
        raw = np.ascontiguousarray(arr).tobytes()
        off = sum(len(c) for c in chunks)
        chunks.append(raw + b"\0" * ((-len(raw)) % 4))
        views.append({"buffer": 0, "byteOffset": off, "byteLength": len(raw)})
        n = int(np.asarray(arr).size) if atype == "SCALAR" else len(arr)
        a = {"bufferView": len(views) - 1, "componentType": ctype, "count": n, "type": atype}
        if atype == "VEC3" and ctype == 5126:
            a["min"], a["max"] = np.asarray(arr).min(0).tolist(), np.asarray(arr).max(0).tolist()
        accessors.append(a)
        return len(accessors) - 1
    quad = np.float32([[-0.5, -0.5, 0], [0.5, -0.5, 0], [0.5, 0.5, 0], [-0.5, 0.5, 0]])
    a_pos = add(quad, 5126, "VEC3")
    a_nrm = add(np.tile(np.float32([0, 0, 1]), (4, 1)), 5126, "VEC3")
    a_uv = add(np.float32([[0, 1], [1, 1], [1, 0], [0, 0]]), 5126, "VEC2")
    a_idx = add(np.uint16([0, 1, 2, 0, 2, 3]), 5123, "SCALAR")
    a_dz = add(np.float32([[0, 0, 0], [0, 0, 0], [0.2, 0.1, 0.4], [0, 0, 0]]), 5126, "VEC3")
    attrs = {"POSITION": a_pos, "NORMAL": a_nrm, "TEXCOORD_0": a_uv}
    samplers, channels = [], []
    for k, (pointer, mode, atype, keys, out) in enumerate(CHANNELS):
        samplers.append({"input": add(np.float32(keys), 5126, "SCALAR"), "output": add(np.float32(out), 5126, atype), "interpolation": mode})
        target = {"path": "pointer"}
        if pointer is not None:
            target["extensions"] = {"KHR_animation_pointer": {"pointer": pointer}}
        channels.append({"sampler": k, "target": target})
    samplers.append({"input": add(np.float32(K3), 5126, "SCALAR"), "output": add(np.float32([[0, 0.9, 0.2], [0.4, 1.1, 0.3], [-0.3, 0.8, 0.1]]), 5126, "VEC3")})
    channels.append({"sampler": len(samplers) - 1, "target": {"node": MOVER, "path": "translation"}})
    samplers.append({"input": add(np.float32(K3), 5126, "SCALAR"), "output": add(np.float32([0.0, 1.0, 0.3]), 5126, "SCALAR")})
    channels.append({"sampler": len(samplers) - 1, "target": {"node": MOVER, "path": "weights"}})
    blob = b"".join(chunks)
    return {
        "asset": {"version": "2.0"},
        "extensionsUsed": ["KHR_animation_pointer", "KHR_lights_punctual", "KHR_node_visibility", "KHR_texture_transform",
                           "KHR_materials_emissive_strength", "KHR_materials_transmission"],
        "extensions": {"KHR_lights_punctual": {"lights": [{"type": "spot", "color": [1.0, 0.9, 0.8], "intensity": 5.0, "range": 10.0,
                                                           "spot": {"innerConeAngle": 0.2, "outerConeAngle": 0.6}}]}},
        "buffers": [{"byteLength": len(blob), "uri": "data:application/octet-stream;base64," + base64.b64encode(blob).decode()}],
        "bufferViews": views, "accessors": accessors,
        "images": [{"uri": _png_data_uri()}], "textures": [{"source": 0}],
        "materials": [
            {"pbrMetallicRoughness": {"baseColorFactor": [0.8, 0.7, 0.6, 1.0], "roughnessFactor": 0.6, "metallicFactor": 0.1},
             "emissiveFactor": [0.1, 0.0, 0.0], "extensions": {"KHR_materials_emissive_strength": {"emissiveStrength": 2.0}}},
            {"alphaMode": "MASK", "alphaCutoff": 0.5, "doubleSided": True,
             "pbrMetallicRoughness": {"metallicFactor": 0.0, "baseColorTexture": {"index": 0, "extensions": {
                 "KHR_texture_transform": {"offset": [0.1, 0.2], "scale": [2.0, 3.0], "rotation": 0.3}}}}},
            {"pbrMetallicRoughness": {"roughnessFactor": 0.1, "metallicFactor": 0.0},
             "extensions": {"KHR_materials_transmission": {"transmissionFactor": 0.0, "transmissionTexture": {"index": 0}}}}],
        "meshes": [{"primitives": [{"attributes": attrs, "indices": a_idx, "material": m}]} for m in (0, 1, 2, 0)] +
                  [{"primitives": [{"attributes": attrs, "indices": a_idx, "material": 0, "targets": [{"POSITION": a_dz}]}], "weights": [0.0]}],
        "cameras": [{"type": "perspective", "perspective": {"yfov": 0.8, "znear": 0.1, "zfar": 100.0}}],
        "nodes": [{"camera": 0, "translation": [0, 0, 4.0]},
                  {"extensions": {"KHR_lights_punctual": {"light": 0}}, "translation": [0.3, 0.5, 3.0]},
                  {"mesh": 0, "translation": [0, 0, -1.0], "scale": [4.0, 3.0, 1.0]},
                  {"mesh": 1, "translation": [-0.9, 0, 0]},
                  {"mesh": 2, "translation": [0.9, 0, 0.5]},
                  {"children": [6]},
                  {"mesh": 3, "translation": [0, -0.9, 0.2], "scale": [0.6, 0.6, 1.0]},
                  {"mesh": 4, "translation": [0, 0.9, 0.2], "scale": [0.6, 0.6, 1.0]}],
        "scenes": [{"nodes": [0, 1, 2, 3, 4, 5, 7]}], "scene": 0,
        "animations": [{"name": "pointers", "samplers": samplers, "channels": channels}],
    }


def write_asset(path, doc=None):
    path.write_text(json.dumps(asset_doc() if doc is None else doc))
    return str(path)


# ---- (a) the float64 restatement of the sampler ---------------------------------------------------------------------------
def _ref_value(mode, atype, keys, out, time):
    """processAnimationChannel + calculateInterpolationFactor + the pointer branches of handle*Interpolation in float64, on the
    fp32 key times and the fp32 time.  Returns (value, bound) or None where the reference applies nothing."""
    keys = np.float32(keys)
    time = np.float32(time)
    k = int(np.searchsorted(keys, time, side="right"))
    if k == 0:
        return None
    i = min(k - 1, len(keys) - 2)
    t0, t1 = float(keys[i]), float(keys[i + 1])
    if time < t0 or time > t1:
        return None
    d = t1 - t0
    t = 0.0 if abs(d) < EPS else min(max((float(time) - t0) / d, 0.0), 1.0)
    o = np.asarray(np.float32(out), np.float64)
    if atype == "SCALAR":
        o = o.reshape(-1)
    if mode == "STEP":
        return o[i], 0.0
    if mode == "CUBICSPLINE":
        if atype == "SCALAR":
            return None
        v0, a, b, v1 = o[3 * i + 1], o[3 * i + 3], o[3 * i + 2], o[3 * i + 4]
        h = (2 * t ** 3 - 3 * t ** 2 + 1, d * (t ** 3 - t ** 2), d * (t ** 3 - 2 * t ** 2 + t), -2 * t ** 3 + 3 * t ** 2)
        return h[0] * v0 + h[1] * a + h[2] * b + h[3] * v1, 32 * EPS * (np.abs(v0) + np.abs(v1) + d * (np.abs(a) + np.abs(b)))
    x, y = o[i], o[i + 1]
    return x * (1 - t) + y * t, 8 * EPS * (np.abs(x) + np.abs(y))


def _get(shadow, pointer):
    from vk_gltf_renderer_b200.animation import _MISSING, _json_get
    v = _json_get(shadow, pointer[1:].split("/"))
    return None if v is _MISSING else v


# ---- (b) the static asset, by hand -------------------------------------------------------------------------------------------
def _static_doc(doc, values):
    """the asset with the sampled values written in: `values` maps pointer -> sampled value for the channels active now"""
    d = copy.deepcopy(doc)
    m0, m1, m2 = d["materials"]
    light = d["extensions"]["KHR_lights_punctual"]["lights"][0]
    for p, v in values.items():
        if p == "/materials/0/pbrMetallicRoughness/baseColorFactor":
            m0["pbrMetallicRoughness"]["baseColorFactor"] = v
        elif p == "/materials/0/pbrMetallicRoughness/roughnessFactor":
            m0["pbrMetallicRoughness"]["roughnessFactor"] = v
        elif p == "/materials/1/alphaCutoff":
            m1["alphaCutoff"] = v
        elif p == "/materials/0/emissiveFactor":
            m0["emissiveFactor"] = v
        elif p.startswith("/materials/1/pbrMetallicRoughness/baseColorTexture/"):
            # a texture-info extension is REPLACED: the asset's scale and rotation are gone
            m1["pbrMetallicRoughness"]["baseColorTexture"]["extensions"]["KHR_texture_transform"] = {"offset": v}
        elif p.startswith("/materials/0/extensions/KHR_materials_emissive_strength/"):
            m0["extensions"]["KHR_materials_emissive_strength"]["emissiveStrength"] = v
        elif p.startswith("/materials/2/extensions/KHR_materials_transmission/"):
            # a material extension is MERGED: its transmissionTexture stays
            m2["extensions"]["KHR_materials_transmission"]["transmissionFactor"] = v
        elif p.startswith(LIGHT):
            key = p[len(LIGHT):]
            if key.startswith("spot/"):
                light["spot"][key[5:]] = v
            else:
                light[key] = v
        elif p == "/nodes/5/extensions/KHR_node_visibility/visible":
            d["nodes"][PARENT]["extensions"] = {"KHR_node_visibility": {"visible": v}}
    return d


def _description(scn):
    return dict(materials=[bytes(m) for m in scn.materials], texture_infos=[bytes(t) for t in scn.texture_infos],
                lights=[bytes(l) for l in scn.lights], visible=[rn["visible"] for rn in scn.render_nodes],
                nodes=[bytes(np.asarray(rn["objectToWorld"], np.float32)) for rn in scn.render_nodes])


def _oracle_image(oracle_mod, scn, env):
    o = oracle_mod.Oracle()
    o.set_scene(scn)
    o.set_environment(env)
    img = oracle_mod.render(o, scn.camera, 48, 36, 2, max_depth=4)
    o.close()
    return img


def test_pointer_channels_sample_and_merge_like_the_reference(tmp_path, oracle_mod, std_env):
    from vk_gltf_renderer_b200 import animation as anim, scene
    doc = asset_doc()
    scn = scene.load_gltf(write_asset(tmp_path / "pointer.gltf", doc))
    loaded = scene.load_gltf(str(tmp_path / "pointer.gltf"))
    an = scn.graph["animations"][0]
    assert [c["pointer"] for c in an["channels"][:len(CHANNELS)]] == [p or "" for p, *_ in CHANNELS]
    assert [s["type"] for s in an["samplers"][:len(CHANNELS)]] == [t for _, _, t, _, _ in CHANNELS]
    assert len(scn.lights) == 1 and scn.light_sources[0][0] == 0
    yfov = scn.camera.yfov
    seen_vis = set()
    for time in TIMES:                               # one scene, every time in turn: nothing may carry over from the last call
        shadow, dirty = anim.sample_pointers(scn, 0, time)
        # (a) values
        values = {}
        for pointer, mode, atype, keys, out in CHANNELS:
            ref = _ref_value(mode, atype, keys, out, time)
            if pointer is None:
                continue
            got = _get(shadow, pointer)
            if ref is None or "01x" in pointer:         # nlohmann refuses "01x" as an index of the array "/materials/0/" made
                assert got is None, (time, pointer, got)
                continue
            v, bound = ref
            if pointer.endswith("/visible"):
                assert got is bool(v != 0), (time, pointer, got)
            else:
                assert np.all(np.abs(np.asarray(got, np.float64) - v) <= bound), (time, pointer, got, v, bound)
            values[pointer] = got
        active = bool(values)
        assert dirty["materials"] == ({0, 1, 2, 9} if active else set()), (time, dirty)    # 01x and /foo/ mark nothing
        assert dirty["lights"] == ({0} if active else set()) and dirty["cameras"] == ({0} if active else set())
        assert dirty["nodes"] == ({PARENT, CHILD} if active else set())
        # (b) the description against the static asset
        anim.apply_pointers(scn, shadow, dirty)
        static = scene.load_gltf(write_asset(tmp_path / "static.gltf", _static_doc(doc, values)))
        assert _description(scn) == _description(static), time
        seen_vis.add(tuple(rn["visible"] for rn in scn.render_nodes))
        assert scn.camera.yfov == yfov                  # the reference writes the camera into its model; no frame reads it
        locals_, _ = anim.sample_animation(scn, 0, time)
        assert np.array_equal(locals_[CHILD], scn.graph["locals"][CHILD])      # the pointer to its translation changes nothing
        # (c) the oracle's image
        assert np.array_equal(_oracle_image(oracle_mod, scn, std_env).view(np.uint32),
                              _oracle_image(oracle_mod, static, std_env).view(np.uint32)), time
    assert len(seen_vis) == 2                           # the parent's child was hidden at some times and shown at others
    # back to a time outside every key range: the loaded description
    anim.apply_pointers(scn, *anim.sample_pointers(scn, 0, 9.0))
    assert _description(scn) == _description(loaded)


def test_pointer_channel_edge_cases(tmp_path):
    """resource indices as std::from_chars parses them, JSON pointers as nlohmann builds them (an array for a first "0" token),
    a VEC2 value on a "/visible" pointer stored as an array, a scene without a glTF document refused"""
    from vk_gltf_renderer_b200 import animation as anim, scene
    assert anim._resource("/materials/3/x") == ("materials", 3)
    assert anim._resource("/materials/01/x") == ("materials", 1)
    assert anim._resource("/materials/01x/x") == ("materials", -1)
    assert anim._resource("/materials/-2/x") == ("materials", -2)
    assert anim._resource("/materials//x") == ("materials", -1)
    assert anim._resource("/nodes/4") == ("nodes", 4)
    assert anim._resource("/foo/0") == (None, -1)
    assert anim._tokens("") is None and anim._tokens("materials/0") is None and anim._tokens("/a~2b") is None
    assert anim._tokens("/a~1b/c~0d") == ["a/b", "c~d"]
    root = {}
    assert anim._json_set(root, ["materials", "0", "x"], 1.0) and root == {"materials": [{"x": 1.0}]}
    assert anim._json_set(root, ["materials", "2", "x"], 2.0) and root["materials"][1] is None
    assert not anim._json_set(root, ["materials", "01", "x"], 3.0)
    assert not anim._json_set(root, ["materials", "2", "x", "y"], 3.0)     # x is a number
    with pytest.raises(ValueError):
        anim.apply_pointers(scene.Scene(), {}, {"materials": set(), "lights": set(), "cameras": set(), "nodes": set()})
