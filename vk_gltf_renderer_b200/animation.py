"""Host side of the animation feed (include/b200pt.h: b200pt_set_animation / b200pt_animate).

Mirrors what SceneAnimationVk prepares for the morph / skinning compute shaders
(src/gltf_scene_animation_vk.cpp:120-260 static task data, :396-494 per-frame data): the task records and the per-frame
joint / normal matrices.  The vertex work itself runs on the device (csrc/animate.cuh); nothing here touches vertices.
The KHR_animation_pointer channels (AnimationPointerSystem) are sampled and merged into the scene description here too
(sample_pointers / apply_pointers); PathTracer.update_scene_changes pushes what they change.
"""
import copy
import re
from dataclasses import dataclass
from typing import Optional

import numpy as np


@dataclass
class MorphTask:
    """one morphed render primitive (MorphResult + MorphGpuData, gltf_scene_animation_vk.cpp:262-330): base arrays and
    per-target deltas [numTargets, vertexCount, 3]"""
    render_prim: int
    base_positions: np.ndarray
    position_deltas: np.ndarray
    base_normals: Optional[np.ndarray] = None
    base_tangents: Optional[np.ndarray] = None
    normal_deltas: Optional[np.ndarray] = None
    tangent_deltas: Optional[np.ndarray] = None
    mesh: int = -1       # glTF mesh whose `weights` drive the targets (cmdUpdateAnimation :440-458)


@dataclass
class SkinTask:
    """one skinned render primitive (SkinTask + SkinGpuData, gltf_scene_animation_vk.cpp:170-226): base arrays, WEIGHTS_0 [V,4],
    JOINTS_0 [V,4] (int32), the skin's joint count"""
    render_prim: int
    base_positions: np.ndarray
    weights: np.ndarray
    joints: np.ndarray
    num_joints: int
    base_normals: Optional[np.ndarray] = None
    base_tangents: Optional[np.ndarray] = None
    skin: int = -1       # glTF skin index (SkinTask::skinID) and the mesh node the joints are expressed against (refNodeID)
    ref_node: int = -1


def joint_matrices(node_world, joint_nodes, inverse_bind, ref_node):
    """Per-frame skin matrices as cmdUpdateAnimation computes them (gltf_scene_animation_vk.cpp:470-484):
        jointMat[i]  = inverse(world[refNode]) * world[joint_i] * inverseBind[i]   (identity when the skin has fewer)
        normalMat[i] = transpose(inverse(mat3(jointMat[i])))
    node_world / inverse_bind: mathematical 4x4 matrices (row, column).  Returns (jointMats [J,4,4], normalMats [J,3,3]) in the
    glm byte order the C-ABI takes: element [j, c, r] = column c, row r.  (The reference evaluates these few products with glm in
    fp32; here they are evaluated in fp64 and rounded once -- the kernels take whatever matrices the host hands them.)"""
    inv_ref = np.linalg.inv(np.asarray(node_world[ref_node], np.float64))
    jm, nm = [], []
    for i, jn in enumerate(joint_nodes):
        ib = np.asarray(inverse_bind[i], np.float64) if i < len(inverse_bind) else np.eye(4)
        m = inv_ref @ np.asarray(node_world[jn], np.float64) @ ib
        jm.append(m.T)                               # column-major bytes
        nm.append(np.linalg.inv(m[:3, :3]))         # transpose(inverse(m3)) stored column-major: element [c, r] = inverse[c, r]
    return np.asarray(jm, np.float32), np.asarray(nm, np.float32)


def topo_levels(parents):
    """BFS levels of a node forest: (topoNodeOrder int32[numNodes], levelOffsets uint32[numLevels + 1]) -- what the reference
    uploads for world_matrix_propagate.comp.slang (one dispatch per level, parents always in an earlier level)."""
    parents = np.asarray(parents, np.int64)
    depth = np.full(len(parents), -1, np.int64)
    for n in range(len(parents)):
        chain = []
        k = n
        while depth[k] < 0 and parents[k] >= 0:
            chain.append(k)
            k = parents[k]
            if len(chain) > len(parents):
                raise ValueError("node hierarchy has a cycle")
        if depth[k] < 0:
            depth[k] = 0
        d = depth[k]
        for c in reversed(chain):
            d += 1
            depth[c] = d
    order = np.argsort(depth, kind="stable").astype(np.int32)
    counts = np.bincount(depth, minlength=int(depth.max()) + 1)
    offsets = np.concatenate([[0], np.cumsum(counts)]).astype(np.uint32)
    return order, offsets


# ---- what the loader's scene graph yields (vk_gltf_renderer_b200.scene.load_gltf fills Scene.graph / morph_prims / skin_prims) ----------
def tasks_from_scene(scn):
    """AnimationSystem::parseMorphTargets / parseSkinTasks (src/gltf_scene_animation.cpp:150-262, 270-316): one MorphTask per render
    primitive with morph targets (base normals / tangents only when a target moves them), one SkinTask per UNIQUE skinned render
    primitive (first render node wins), with the static base arrays taken from the primitive as loaded."""
    morphs, skins = [], []
    for pid, mp in sorted(scn.morph_prims.items()):
        prim = scn.render_prims[pid]
        morphs.append(MorphTask(pid, prim["positions"].copy(), mp["position_deltas"], mesh=mp["mesh"],
                                base_normals=prim["normals"].copy() if (mp["normal_deltas"] is not None and prim["normals"] is not None) else None,
                                base_tangents=prim["tangents"].copy() if (mp["tangent_deltas"] is not None and prim["tangents"] is not None) else None,
                                normal_deltas=mp["normal_deltas"], tangent_deltas=mp["tangent_deltas"]))
    seen = set()
    for rn, (node_id, skin_id, _) in zip(scn.render_nodes, scn.graph["render_nodes"] if scn.graph else []):
        pid = rn["renderPrimID"]
        if skin_id < 0 or pid in seen or pid not in scn.skin_prims or skin_id >= len(scn.graph["skins"]):
            continue
        seen.add(pid)
        prim, sp = scn.render_prims[pid], scn.skin_prims[pid]
        skins.append(SkinTask(pid, prim["positions"].copy(), sp["weights"], sp["joints"], len(scn.graph["skins"][skin_id]["joints"]),
                              base_normals=None if prim["normals"] is None else prim["normals"].copy(),
                              base_tangents=None if prim["tangents"] is None else prim["tangents"].copy(), skin=skin_id, ref_node=node_id))
    return morphs, skins


def node_hierarchy(scn):
    """(parents, RenderNodeGpuMapping triples, instance matrices [R,4,4] glm-ordered) for PathTracer.set_node_hierarchy"""
    g = scn.graph
    mappings = [(node_id, rn["materialID"], rn["renderPrimID"]) for rn, (node_id, _, _) in zip(scn.render_nodes, g["render_nodes"])]
    inst = np.ascontiguousarray(np.asarray([lm for _, _, lm in g["render_nodes"]], np.float64).reshape(-1, 4, 4).transpose(0, 2, 1).astype(np.float32))
    return g["parents"], mappings, inst


def world_matrices(parents, locals_):
    """fp64 world matrices of the node graph (the host's view; the device propagates its own in fp32)"""
    locals_ = np.asarray(locals_, np.float64)
    world = [None] * len(parents)

    def get(n):
        if world[n] is None:
            world[n] = locals_[n] if parents[n] < 0 else get(int(parents[n])) @ locals_[n]
        return world[n]
    return np.asarray([get(n) for n in range(len(parents))])


def frame_inputs(scn, morph_tasks, skin_tasks, locals_=None, mesh_weights=None):
    """The per-frame data of one cmdUpdateAnimation (src/gltf_scene_animation_vk.cpp:430-494) for the given node-local matrices
    (default: the asset's rest pose) and mesh weights (default: mesh.weights): morph weights per morph task, joint / normal matrices per
    skin task.  sample_animation samples an animation's channels into those locals / weights; its KHR_animation_pointer channels
    go through sample_pointers / apply_pointers and PathTracer.update_scene_changes instead."""
    g = scn.graph
    world = world_matrices(g["parents"], g["locals"] if locals_ is None else locals_)
    weights = []
    for t in morph_tasks:
        w = (mesh_weights or {}).get(t.mesh, g["mesh_weights"].get(t.mesh, np.zeros(0, np.float32)))
        full = np.zeros(t.position_deltas.shape[0], np.float32)          # fewer weights than targets: the rest stay 0 (:446-452)
        full[:min(len(w), len(full))] = np.asarray(w, np.float32)[:len(full)]
        weights.append(full)
    jms, nms = [], []
    for t in skin_tasks:
        sk = g["skins"][t.skin]
        ibm = [] if sk["ibm"] is None else list(sk["ibm"])
        jm, nm = joint_matrices(world, sk["joints"], ibm, t.ref_node)
        jms.append(jm)
        nms.append(nm)
    return weights, jms, nms


# ---- the caller of the feed: sampling an animation into node-local matrices and mesh weights ---------------------------------------
def _slerp(q1, q2, t):
    """glm::slerp(x, y, a) on (x, y, z, w) quaternions: shortest path, linear blend when the two are (nearly) parallel"""
    q1, q2 = np.asarray(q1, np.float64), np.asarray(q2, np.float64)
    c = float(np.dot(q1, q2))
    if c < 0.0:
        q2, c = -q2, -c
    if c > 1.0 - 1.1920929e-07:
        return q1 + (q2 - q1) * t
    ang = np.arccos(c)
    return (np.sin((1.0 - t) * ang) * q1 + np.sin(t * ang) * q2) / np.sin(ang)


def _cubic(values, t, key_delta, index):
    """computeCubicInterpolation (src/gltf_scene_animation.cpp:498-517): glTF Hermite spline over [in-tangent, value, out-tangent] triplets"""
    t2, t3 = t * t, t * t * t
    c_v1 = -2 * t3 + 3 * t2
    c_v0 = 1 - c_v1
    c_a = key_delta * (t3 - t2)
    c_b = key_delta * (t3 - 2 * t2 + t)
    prev, nxt = index * 3, (index + 1) * 3
    return values[prev + 1] * c_v0 + values[nxt + 0] * c_a + values[prev + 2] * c_b + values[nxt + 1] * c_v1


def sample_animation(scn, animation=0, time=0.0):
    """AnimationSystem::updateAnimation / processAnimationChannel (src/gltf_scene_animation.cpp:352-479) evaluated from the asset's rest
    pose: every translation / rotation / scale / weights channel whose keyframe range contains `time` overwrites its node's value --
    LINEAR (slerp for rotations, :530-583), STEP (:598-628; weights are left alone there) and CUBICSPLINE (:640-688; rotation
    re-normalised) -- then the node-local matrices are rebuilt (T * R * S; a node given as a matrix and not animated keeps it).
    KHR_animation_pointer channels of the same animation are sampled by sample_pointers and applied by apply_pointers; a pointer
    to a node's translation / rotation / scale / weights is not read here, as in the reference.
    Returns (locals f64 [N, 4, 4], mesh_weights {mesh: f32[T]}) for frame_inputs / PathTracer.update_node_matrices."""
    from .scene import _trs
    g = scn.graph
    trs = [dict(t) for t in g["trs"]]
    weights = {m: w.copy() for m, w in g["mesh_weights"].items()}
    animated = set()
    if 0 <= animation < len(g["animations"]):
        an = g["animations"][animation]
        for ch in an["channels"]:
            node, path = ch["node"], ch["path"]
            if not (0 <= node < len(trs)) or path not in ("translation", "rotation", "scale", "weights"):
                continue
            sm = an["samplers"][ch["sampler"]]
            inp = sm["inputs"]
            if len(inp) < 2:
                continue
            k = int(np.searchsorted(inp, np.float32(time), side="right"))     # first key strictly after `time`
            if k == 0:
                continue
            i = min(k - 1, len(inp) - 2)
            t0, t1 = float(inp[i]), float(inp[i + 1])
            if time < t0 or time > t1:
                continue
            dt = t1 - t0
            f = 0.0 if abs(dt) < 1.1920929e-07 else min(max((time - t0) / dt, 0.0), 1.0)
            out = sm["outputs"]
            mode = sm["interpolation"]
            if path == "weights":
                mesh = trs[node]["mesh"]
                if mesh < 0 or mode != "LINEAR":
                    continue
                nt = out.size // len(inp)
                o = out.reshape(len(inp), nt)
                weights[mesh] = ((1.0 - f) * o[i] + f * o[i + 1]).astype(np.float32)
                continue
            o = out.reshape(-1, 4 if path == "rotation" else 3).astype(np.float64)
            if mode == "STEP":
                v = o[i]
            elif mode == "CUBICSPLINE":
                if len(o) <= (i + 1) * 3 + 1:
                    continue
                v = _cubic(o, f, dt, i)
                if path == "rotation":
                    v = v / np.linalg.norm(v)
            else:
                if path == "rotation":
                    v = _slerp(o[i], o[i + 1], f)
                    v = v / np.linalg.norm(v)
                else:
                    v = (1.0 - f) * o[i] + f * o[i + 1]
            trs[node][path] = v.tolist()
            animated.add(node)
    locals_ = g["locals"].copy()
    for n in animated:
        t = trs[n]
        locals_[n] = _trs(np.asarray(t["translation"], np.float64), np.asarray(t["rotation"], np.float64), np.asarray(t["scale"], np.float64))
    return locals_, weights


# ---- KHR_animation_pointer: AnimationPointerSystem (src/gltf_animation_pointer.cpp) and its merge into the scene -------------------
_F32 = np.float32
_FLT_EPSILON = np.finfo(np.float32).eps
# parseResourceInfo's prefixes (gltf_animation_pointer.cpp:114-117) and the key of each kind in sample_pointers' dirty sets
_RESOURCES = (("/materials/", "materials"), ("/extensions/KHR_lights_punctual/lights/", "lights"), ("/cameras/", "cameras"),
              ("/nodes/", "nodes"))
_FROM_CHARS_INT = re.compile(r"-?[0-9]+")
_ARRAY_INDEX = re.compile(r"0|[1-9][0-9]*")


def _resource(pointer):
    """parseResourceInfo (gltf_animation_pointer.cpp:103-139): (kind, index) of a pointer.  The token after the prefix must parse
    completely as an int (std::from_chars), else the index is -1; an unknown prefix gives kind None."""
    for prefix, kind in _RESOURCES:
        if pointer.startswith(prefix):
            tok = pointer[len(prefix):].split("/", 1)[0]
            ok = _FROM_CHARS_INT.fullmatch(tok) is not None and -2 ** 31 <= int(tok) < 2 ** 31
            return kind, int(tok) if ok else -1
    return None, -1


def _tokens(pointer):
    """the reference tokens of nlohmann::json_pointer(pointer), None where its constructor throws (no leading '/', a '~' not
    followed by 0 or 1).  The empty pointer, which nlohmann reads as the whole document, is None too: a pointer channel without
    the extension changes nothing."""
    if not pointer.startswith("/"):
        return None
    toks = pointer[1:].split("/")
    if any(re.search(r"~(?![01])", t) for t in toks):
        return None
    return [t.replace("~1", "/").replace("~0", "~") for t in toks]


def _json_set(root, toks, value):
    """m_jsonModel[json_pointer] = value: missing levels are created (an array when the token is "0", else an object), arrays grow
    with nulls; False where nlohmann throws (a token that is not an array index, a level that is a number or a bool)"""
    holder, key = [root], 0
    for tok in toks:
        cur = holder[key]
        if cur is None:
            cur = holder[key] = [] if tok == "0" else {}
        if isinstance(cur, dict):
            cur.setdefault(tok, None)
            holder, key = cur, tok
        elif isinstance(cur, list):
            if not _ARRAY_INDEX.fullmatch(tok):
                return False
            idx = int(tok)
            cur.extend([None] * (idx + 1 - len(cur)))
            holder, key = cur, idx
        else:
            return False
    holder[key] = value
    return True


_MISSING = object()


def _json_get(root, toks):
    """m_jsonModel.at(json_pointer), _MISSING where it throws"""
    cur = root
    for tok in toks:
        if isinstance(cur, dict) and tok in cur:
            cur = cur[tok]
        elif isinstance(cur, list) and _ARRAY_INDEX.fullmatch(tok) and int(tok) < len(cur):
            cur = cur[int(tok)]
        else:
            return _MISSING
    return cur


def _pointer_value(sm, i, t, key_delta):
    """handleLinearInterpolation / handleStepInterpolation / handleCubicSplineInterpolation for a pointer channel
    (gltf_scene_animation.cpp:570-583, 620-628, 646-657): the value of key segment i at factor t by the output accessor's type, or
    None where the reference applies nothing.  A SCALAR sampler uses element 0 of each key's elements and has no CUBICSPLINE."""
    kind, mode, out, n = sm["type"], sm["interpolation"], sm["outputs"], len(sm["inputs"])
    if kind == "SCALAR":
        per = out.size // n
        if per == 0 or mode == "CUBICSPLINE":
            return None
        o = out.reshape(-1)[:n * per].reshape(n, per)[:, 0]
    elif kind in ("VEC2", "VEC3", "VEC4"):
        o = out.reshape(-1, int(kind[-1]))
    else:
        return None
    if mode == "STEP":
        return o[i] if i < len(o) else None
    if mode == "CUBICSPLINE":
        return _cubic(o, t, key_delta, i) if len(o) > (i + 1) * 3 + 1 else None
    return o[i] * (_F32(1) - t) + o[i + 1] * t if i + 1 < len(o) else None      # glm::mix


def sample_pointers(scn, animation=0, time=0.0):
    """The KHR_animation_pointer half of AnimationSystem::updateAnimation (src/gltf_scene_animation.cpp:377-380) evaluated from the
    loaded asset: every "pointer" channel whose keyframe range contains `time` writes its value into a sparse JSON of the animated
    values (AnimationPointerSystem::applyValue, gltf_animation_pointer.cpp:146-235), and the resource its pointer names is marked
    dirty when the index parses and the prefix is known.  Keys and factor as processAnimationChannel / calculateInterpolationFactor:
    upper_bound on the fp32 time, the last segment clamped, 0 on a segment shorter than FLT_EPSILON, clamped to [0, 1].  Values are
    evaluated in fp32 in the reference's operation order without fused multiply-adds (glm::mix x * (1 - t) + y * t; the Hermite
    form of computeCubicInterpolation); whether the reference's compiler contracts those products is unpinned.  A pointer ending in
    "/visible" stores value != 0.
    The reference keeps its JSON across frames, so a channel outside its key range keeps its last value there; here every call
    starts from the loaded asset, so such a channel shows the loaded value (DESIGN.md §4).
    Returns (shadow JSON dict, {"materials" | "lights" | "cameras" | "nodes": set of indices}) for apply_pointers."""
    shadow, dirty = {}, {kind: set() for _, kind in _RESOURCES}
    g = scn.graph
    if g is None or not 0 <= animation < len(g["animations"]):
        return shadow, dirty
    an = g["animations"][animation]
    time = _F32(time)
    for ch in an["channels"]:
        if ch["path"] != "pointer" or not 0 <= ch["sampler"] < len(an["samplers"]):
            continue
        sm = an["samplers"][ch["sampler"]]
        inp = sm["inputs"]
        if len(inp) < 2:
            continue
        k = int(np.searchsorted(inp, time, side="right"))
        if k == 0:
            continue
        i = min(k - 1, len(inp) - 2)
        t0, t1 = inp[i], inp[i + 1]
        if time < t0 or time > t1:
            continue
        key_delta = t1 - t0
        t = _F32(0) if abs(key_delta) < _FLT_EPSILON else min(max((time - t0) / key_delta, _F32(0)), _F32(1))
        v = _pointer_value(sm, i, t, key_delta)
        toks = _tokens(ch["pointer"])
        if v is None or toks is None:
            continue
        if np.ndim(v) == 0:
            v = bool(v != 0) if ch["pointer"].endswith("/visible") else float(v)
        else:
            v = [float(x) for x in v]
        if _json_set(shadow, toks, v):
            kind, idx = _resource(ch["pointer"])
            if kind is not None and idx >= 0:
                dirty[kind].add(idx)
    return shadow, dirty


class _JsonTypeError(Exception):
    """nlohmann::json::type_error: a sync stops at the value it cannot read and keeps what it merged before"""


def _f(v):
    """json::get<double>(): numbers and booleans"""
    if isinstance(v, (bool, float)):
        return float(v)
    raise _JsonTypeError


def _set_elems(d, key, default, arr, n):
    cur = list(d.get(key, default))
    d[key] = cur
    for i in range(n):
        cur[i] = _f(arr[i])


def _replace_extensions(js, parent, key):
    """mergeExtensions (gltf_animation_pointer.cpp:479-488): each extension the JSON names REPLACES the asset's"""
    if isinstance(js, dict) and isinstance(js.get("extensions"), dict):
        ext = parent.setdefault(key, {}).setdefault("extensions", {})
        for name, v in js["extensions"].items():
            ext[name] = copy.deepcopy(v)


def _deep_merge(parent, key, src):
    """mergeValue (gltf_animation_pointer.cpp:38-63)"""
    tgt = parent[key]
    if not isinstance(src, dict) or not isinstance(tgt, dict):
        parent[key] = copy.deepcopy(src)
        return
    for k, v in src.items():
        if k in tgt and isinstance(v, dict) and isinstance(tgt[k], dict):
            _deep_merge(tgt, k, v)
        else:
            tgt[k] = copy.deepcopy(v)


def _merge_material_fields(m, js):
    """mergeJsonIntoMaterial (gltf_animation_pointer.cpp:474-577) on the glTF JSON of one material"""
    if not isinstance(js, dict):
        return
    pj = js.get("pbrMetallicRoughness")
    if isinstance(pj, dict):
        pbr = m.setdefault("pbrMetallicRoughness", {})
        for k in ("roughnessFactor", "metallicFactor"):
            if isinstance(pj.get(k), float):
                pbr[k] = pj[k]
        if isinstance(pj.get("baseColorFactor"), list) and len(pj["baseColorFactor"]) >= 4:
            _set_elems(pbr, "baseColorFactor", [1.0, 1.0, 1.0, 1.0], pj["baseColorFactor"], 4)
        for k in ("baseColorTexture", "metallicRoughnessTexture"):
            if k in pj:
                _replace_extensions(pj[k], pbr, k)
    if isinstance(js.get("emissiveFactor"), list) and len(js["emissiveFactor"]) >= 3:
        _set_elems(m, "emissiveFactor", [0.0, 0.0, 0.0], js["emissiveFactor"], 3)
    if "emissiveTexture" in js:
        _replace_extensions(js["emissiveTexture"], m, "emissiveTexture")
    for k, field in (("normalTexture", "scale"), ("occlusionTexture", "strength")):
        if k in js:
            if isinstance(js[k], dict) and isinstance(js[k].get(field), float):
                m.setdefault(k, {})[field] = js[k][field]
            _replace_extensions(js[k], m, k)
    if isinstance(js.get("alphaCutoff"), float):
        m["alphaCutoff"] = js["alphaCutoff"]
    # (alphaMode and doubleSided take a string and a boolean: no animated value is either)
    if isinstance(js.get("extensions"), dict):
        ext = m.setdefault("extensions", {})
        for name, v in js["extensions"].items():
            if name in ext:
                _deep_merge(ext, name, v)       # material extensions are MERGED: their other keys survive
            else:
                ext[name] = copy.deepcopy(v)


def _merge_light_fields(L, js):
    """syncLight (gltf_animation_pointer.cpp:292-327) on the glTF JSON of one light"""
    if not isinstance(js, dict):
        return
    if isinstance(js.get("color"), list):
        col = (list(L.get("color", [1.0, 1.0, 1.0])) + [0.0] * 3)[:3]
        L["color"] = col
        for i, x in enumerate(js["color"][:3]):
            col[i] = _f(x)
    for k in ("intensity", "range"):
        if k in js:
            L[k] = _f(js[k])
    if isinstance(js.get("spot"), dict):
        spot = L.setdefault("spot", {})
        for k in ("innerConeAngle", "outerConeAngle"):
            if k in js["spot"]:
                spot[k] = _f(js["spot"][k])


def _merged(src, js, merge):
    out = copy.deepcopy(src)
    try:
        merge(out, js)
    except _JsonTypeError:
        pass
    return out


def apply_pointers(scn, shadow, dirty):
    """AnimationPointerSystem::syncToModel (gltf_animation_pointer.cpp:241-397) and the host side of the scene update that follows,
    from the loaded asset: scn.materials / texture_infos are rebuilt from the asset's materials, each dirty one merged with the JSON of
    sample_pointers and put through MaterialCache.updateMaterial (the texture-info slots stay); scn.lights are converted again from
    the asset's lights, dirty ones merged, each with its node's world matrix at load; every node's visibility is the asset's, a
    dirty node's KHR_node_visibility replaced by the JSON's, inherited down the node graph (Scene.set_node_visible).  Nodes take
    nothing else (syncNode: a pointer to translation / rotation / scale / weights changes nothing) and cameras nothing at all (the
    reference writes them into its model, which no frame reads).  Push the result with PathTracer.update_scene_changes."""
    from .scene import MaterialCache, make_light, node_visible
    j = scn.gltf
    if j is None:
        raise ValueError("apply_pointers needs a scene loaded from glTF")
    mats = j.get("materials", [])
    cache = MaterialCache()
    cache.buildFromMaterials(mats or [{}])
    for m in sorted(dirty["materials"]):
        js = _json_get(shadow, ["materials", str(m)])
        if m < len(mats) and js is not _MISSING:
            cache.updateMaterial(m, _merged(mats[m], js, _merge_material_fields))
    scn.materials, scn.texture_infos = cache.getShadeMaterials(), cache.getTextureInfos()
    lights = j.get("extensions", {}).get("KHR_lights_punctual", {}).get("lights", [])
    merged = {}
    for li in dirty["lights"]:
        js = _json_get(shadow, ["extensions", "KHR_lights_punctual", "lights", str(li)])
        if li < len(lights) and js is not _MISSING:
            merged[li] = _merged(lights[li], js, _merge_light_fields)
    scn.lights = [make_light(merged.get(li, lights[li]), world) for li, world in scn.light_sources]
    nodes = j.get("nodes", [])
    scn.node_visible = [node_visible(n) for n in nodes]
    for n in dirty["nodes"]:
        js = _json_get(shadow, ["nodes", str(n)])
        if n < len(nodes) and isinstance(js, dict) and isinstance(js.get("extensions"), dict):
            scn.node_visible[n] = node_visible({"extensions": {**nodes[n].get("extensions", {}), **js["extensions"]}})
    scn._apply_visibility()
