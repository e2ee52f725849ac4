"""Minimal glTF 2.0 -> path-tracer scene arrays.

The reference's CPU scene model (src/gltf_scene.cpp, tinygltf) is *consumed*, not rebuilt, by
the hot path (SURVEY.md §2 row 7).  tinygltf/glm are not in this image, so this module produces
the same *outputs* that SceneVk/MaterialCache/SceneRtx hand the path tracer:

  RenderPrimitive[]   unique (attributes, indices) in mesh/primitive order   gltf_scene.cpp:2139-2163
  RenderNode[]        one per (node, primitive), DFS order, + GPU instancing  gltf_scene.cpp:2338-2429
  GltfShadeMaterial[] + GltfTextureInfo[] (slot 0 reserved)                  gltf_material_cache.cpp:63-251
  vertex arrays       float3 pos/nrm, float2 uv0/uv1, float4 tan, unorm4x8   gltf_scene_vk.cpp:741-869
  GltfLight[]                                                                 gltf_scene_vk.cpp:1354-1394
  textures + samplers + sRGB set                                              gltf_scene_vk.cpp:909-947,1102-1154
  first camera (eye/center/up from node extras or node matrix)               gltf_scene.cpp:2215-2267
"""
import base64
import ctypes as C
import io
import json
import math
import os
import struct

import numpy as np

from . import abi

_COMP = {5120: np.int8, 5121: np.uint8, 5122: np.int16, 5123: np.uint16, 5124: np.int32, 5125: np.uint32, 5126: np.float32}
_NCOMP = {"SCALAR": 1, "VEC2": 2, "VEC3": 3, "VEC4": 4, "MAT2": 4, "MAT3": 9, "MAT4": 16}


class Camera:
    def __init__(self):
        self.type = "perspective"
        self.eye = np.array([0, 0, 1], np.float32)
        self.center = np.zeros(3, np.float32)
        self.up = np.array([0, 1, 0], np.float32)
        self.yfov = math.radians(45.0)
        self.znear = 0.1
        self.zfar = 1000.0
        self.xmag = 1.0
        self.ymag = 1.0


class Scene:
    """Flat scene arrays + the ctypes SceneDesc that points at them."""

    def __init__(self):
        self.render_nodes = []        # list of dict(objectToWorld f32[16] (glm column-major), materialID, renderPrimID, visible)
        self.render_prims = []        # list of dict(indices u32[T,3], positions f32[V,3], normals?, colors?, tangents?, uv0?, uv1?)
        self.materials = []           # list of abi.ShadeMaterial
        self.texture_infos = [abi.TextureInfo()]
        self.texture_infos[0].index = -1
        self.texture_infos[0].uvTransform[:] = [1, 0, 0, 1, 0, 0]
        self.textures = []            # list of dict(rgba8 u8[H,W,4], srgb, wrapS, wrapT, magFilter, minFilter)
        self.lights = []              # list of abi.Light
        # EXT_mesh_opacity_micromap (reference src/gltf_scene_omm.cpp): root micromaps[] and the per-primitive linkage
        self.micromaps = []           # list of dict(data u8[N], triangles abi.MICROMAP_TRIANGLE_DTYPE[M])
        self.prim_omms = []           # list of dict(renderPrimID, micromap, baseTriangle, indices i32[T] | None)
        self.camera = None
        # animation inputs the loader gathers like AnimationSystem::parseMorphTargets / parseSkinTasks (src/gltf_scene_animation.cpp:150-330)
        # and the node graph the GPU transform path consumes; None for scenes built by hand
        self.graph = None             # dict(parents i32[N], locals f64[N,4,4], render_nodes [(nodeID, skinID, instLocal f64[4,4])], skins [dict(joints, ibm)], mesh_weights {mesh: f32[T]})
        self.morph_prims = {}         # renderPrimID -> dict(mesh, position_deltas f32[T,V,3], normal_deltas | None, tangent_deltas | None)
        self.skin_prims = {}          # renderPrimID -> dict(joints i32[V,4], weights f32[V,4])
        # KHR_materials_variants: the root's variant names; a loaded render node carries its primitive's mappings
        # ("variantMaterials": {variant: material}) and its own material ("defaultMaterial")
        self.variants = []
        # KHR_node_visibility: every glTF node's own flag (a loaded scene); a render node is visible when its node and every
        # ancestor are (Scene::traverseSceneWithVisibility)
        self.node_visible = None
        # a loaded scene's glTF document, and per light the glTF light index and the world matrix of its node: what
        # animation.apply_pointers converts again when KHR_animation_pointer channels change materials, lights or nodes
        self.gltf = None
        self.light_sources = []
        self._keep = []

    # -- bounds (reference: Scene::getSceneBounds, gltf_scene.cpp:2303-2336, from transformed vertices)
    def bounds(self):
        lo = np.full(3, np.inf)
        hi = np.full(3, -np.inf)
        for rn in self.render_nodes:
            m = np.asarray(rn["objectToWorld"], np.float64).reshape(4, 4).T
            p = self.render_prims[rn["renderPrimID"]]["positions"].astype(np.float64)
            w = p @ m[:3, :3].T + m[:3, 3]
            lo = np.minimum(lo, w.min(0))
            hi = np.maximum(hi, w.max(0))
        return lo, hi

    def set_variant(self, variant):
        """Scene::setCurrentVariant: every render node takes its primitive's material for `variant` (an index into
        self.variants), or its own material where the primitive maps none; None restores the own materials.  Push the
        result with PathTracer.update_node_materials."""
        for rn in self.render_nodes:
            if "defaultMaterial" in rn:
                rn["materialID"] = rn["variantMaterials"].get(variant, rn["defaultMaterial"])

    def set_node_visible(self, node, visible):
        """KHR_node_visibility of glTF node `node`; the render nodes below it follow (an invisible node hides its whole
        subtree).  Push the result with PathTracer.set_node_visibility."""
        if self.node_visible is None:
            raise ValueError("set_node_visible needs a scene loaded from glTF (its node graph)")
        self.node_visible[node] = bool(visible)
        self._apply_visibility()

    def _apply_visibility(self):
        parents = self.graph["parents"]
        memo = {}

        def shown(n):
            if n not in memo:
                memo[n] = self.node_visible[n] and (parents[n] < 0 or shown(int(parents[n])))
            return memo[n]
        for rn, (nid, _, _) in zip(self.render_nodes, self.graph["render_nodes"]):
            rn["visible"] = shown(nid)

    def num_triangles(self):
        return sum(len(self.render_prims[rn["renderPrimID"]]["indices"]) for rn in self.render_nodes
                   if rn.get("visible", True))

    def add_material(self, **kw):
        m = default_material()
        for k, v in kw.items():
            cur = getattr(m, k)
            if hasattr(cur, "__len__"):
                for i, x in enumerate(v):
                    cur[i] = x
            else:
                setattr(m, k, v)
        self.materials.append(m)
        return len(self.materials) - 1

    def add_texture_info(self, tex_index, texcoord=0, uv_transform=(1, 0, 0, 1, 0, 0)):
        ti = abi.TextureInfo()
        ti.index = tex_index
        ti.texCoord = min(texcoord, 1)
        ti.uvTransform[:] = list(uv_transform)
        self.texture_infos.append(ti)
        return len(self.texture_infos) - 1

    def add_texture(self, rgba8, srgb=False, wrapS=10497, wrapT=10497, magFilter=-1, minFilter=-1):
        rgba8 = np.ascontiguousarray(rgba8, np.uint8)
        assert rgba8.ndim == 3 and rgba8.shape[2] == 4
        self.textures.append(dict(rgba8=rgba8, srgb=int(srgb), wrapS=wrapS, wrapT=wrapT,
                                  magFilter=magFilter, minFilter=minFilter))
        return len(self.textures) - 1

    def add_primitive(self, positions, indices, normals=None, uv0=None, uv1=None, tangents=None, colors=None):
        prim = dict(
            positions=np.ascontiguousarray(positions, np.float32).reshape(-1, 3),
            indices=np.ascontiguousarray(indices, np.uint32).reshape(-1, 3),
            normals=None if normals is None else np.ascontiguousarray(normals, np.float32).reshape(-1, 3),
            uv0=None if uv0 is None else np.ascontiguousarray(uv0, np.float32).reshape(-1, 2),
            uv1=None if uv1 is None else np.ascontiguousarray(uv1, np.float32).reshape(-1, 2),
            tangents=None if tangents is None else np.ascontiguousarray(tangents, np.float32).reshape(-1, 4),
            colors=None if colors is None else np.ascontiguousarray(colors, np.uint32).reshape(-1),
        )
        self.render_prims.append(prim)
        return len(self.render_prims) - 1

    def add_node(self, prim_id, material_id, matrix=None, visible=True):
        m = np.eye(4, dtype=np.float64) if matrix is None else np.asarray(matrix, np.float64).reshape(4, 4)
        self.render_nodes.append(dict(objectToWorld=_glm(m), worldToObject=_glm(np.linalg.inv(m)),
                                      materialID=material_id, renderPrimID=prim_id, visible=visible))
        return len(self.render_nodes) - 1

    def omm_desc(self):
        """(micromaps array, count, primitive linkage array, count, keep-alive) for b200pt_set_opacity_micromaps"""
        keep = []
        mm = (abi.Micromap * max(len(self.micromaps), 1))()
        for i, m in enumerate(self.micromaps):
            data = np.ascontiguousarray(m["data"], np.uint8)
            tris = np.ascontiguousarray(m["triangles"], abi.MICROMAP_TRIANGLE_DTYPE)
            keep += [data, tris]
            mm[i].data = data.ctypes.data_as(abi.c_u8_p)
            mm[i].dataSize = data.size
            mm[i].triangles = tris.ctypes.data_as(C.POINTER(abi.MicromapTriangle))
            mm[i].numTriangles = tris.size
        po = (abi.PrimitiveOmm * max(len(self.prim_omms), 1))()
        for i, p in enumerate(self.prim_omms):
            po[i].renderPrimID, po[i].micromap, po[i].baseTriangle = p["renderPrimID"], p["micromap"], p.get("baseTriangle", 0)
            if p.get("indices") is not None:
                idx = np.ascontiguousarray(p["indices"], np.int32)
                keep.append(idx)
                po[i].indices = idx.ctypes.data_as(C.POINTER(C.c_int32))
                po[i].numIndices = idx.size
        return mm, len(self.micromaps), po, len(self.prim_omms), keep

    # -- ctypes view ---------------------------------------------------------------------------
    def desc(self):
        """Build (and cache) the abi.SceneDesc; arrays stay alive as long as `self` does."""
        keep = []
        n = len(self.render_nodes)
        nodes = (abi.RenderNode * max(n, 1))()
        vis = np.ones(max(n, 1), np.uint8)
        for i, rn in enumerate(self.render_nodes):
            nodes[i].objectToWorld[:] = rn["objectToWorld"].tolist()
            nodes[i].worldToObject[:] = rn["worldToObject"].tolist()
            nodes[i].materialID = rn["materialID"]
            nodes[i].renderPrimID = rn["renderPrimID"]
            vis[i] = 1 if rn.get("visible", True) else 0
        prims = (abi.RenderPrimitive * max(len(self.render_prims), 1))()
        for i, p in enumerate(self.render_prims):
            prims[i].indices = abi.u32ptr(p["indices"])
            prims[i].positions = abi.fptr(p["positions"])
            prims[i].normals = abi.fptr(p["normals"])
            prims[i].colors = abi.u32ptr(p["colors"])
            prims[i].tangents = abi.fptr(p["tangents"])
            prims[i].texCoords[0] = abi.fptr(p["uv0"])
            prims[i].texCoords[1] = abi.fptr(p["uv1"])
            prims[i].triangleCount = len(p["indices"])
            prims[i].vertexCount = len(p["positions"])
        mats = (abi.ShadeMaterial * max(len(self.materials), 1))(*self.materials)
        tis = (abi.TextureInfo * len(self.texture_infos))(*self.texture_infos)
        texs = (abi.Texture * max(len(self.textures), 1))()
        for i, t in enumerate(self.textures):
            texs[i].rgba8 = abi.u8ptr(t["rgba8"])
            texs[i].height, texs[i].width = t["rgba8"].shape[:2]
            for k in ("srgb", "wrapS", "wrapT", "magFilter", "minFilter"):
                setattr(texs[i], k, t[k])
        lights = (abi.Light * max(len(self.lights), 1))(*self.lights)
        d = abi.SceneDesc()
        d.renderNodes, d.numRenderNodes = nodes, n
        d.renderNodeVisible = abi.u8ptr(vis)
        d.renderPrimitives, d.numRenderPrimitives = prims, len(self.render_prims)
        d.materials, d.numMaterials = mats, len(self.materials)
        d.textureInfos, d.numTextureInfos = tis, len(self.texture_infos)
        d.textures, d.numTextures = texs, len(self.textures)
        d.lights, d.numLights = lights, len(self.lights)
        keep += [nodes, vis, prims, mats, tis, texs, lights]
        self._keep = keep
        return d


    # ---- scene blob: what the C++ host (host/b200pt_host.cpp) loads ------------------------------------------
    def save_blob(self, path, env_rgb=None):
        """Serialise the scene (and optionally the HDR environment) into the little-endian "B2SC" blob the C++ host
        reads: the C-ABI structs verbatim plus the attribute arrays.  Stands in for the reference's own loader,
        whose output (SceneVk / MaterialCache arrays) is exactly this data."""
        import struct
        cam = self.camera
        with open(path, "wb") as f:
            f.write(b"B2SC")
            f.write(struct.pack("<7I", 1, len(self.render_nodes), len(self.render_prims), len(self.materials), len(self.texture_infos),
                                len(self.textures), len(self.lights)))
            f.write(struct.pack("<I", 1 if cam.type == "orthographic" else 0))
            f.write(np.asarray(list(cam.eye) + list(cam.center) + list(cam.up) + [cam.yfov, cam.znear, cam.zfar, getattr(cam, "xmag", 1.0),
                                                                                    getattr(cam, "ymag", 1.0)], "<f4").tobytes())
            for rn in self.render_nodes:
                f.write(np.asarray(rn["objectToWorld"], "<f4").tobytes())
                f.write(np.asarray(rn["worldToObject"], "<f4").tobytes())
                f.write(struct.pack("<iiI", rn["materialID"], rn["renderPrimID"], 1 if rn.get("visible", True) else 0))
            for p in self.render_prims:
                names = ("normals", "uv0", "uv1", "tangents", "colors")
                mask = sum(1 << i for i, n in enumerate(names) if p[n] is not None)
                f.write(struct.pack("<3I", len(p["positions"]), len(p["indices"]), mask))
                f.write(np.ascontiguousarray(p["positions"], "<f4").tobytes())
                f.write(np.ascontiguousarray(p["indices"], "<u4").tobytes())
                for n in names:
                    if p[n] is not None:
                        f.write(np.ascontiguousarray(p[n], "<u4" if n == "colors" else "<f4").tobytes())
            for m in self.materials:
                f.write(bytes(m))
            for t in self.texture_infos:
                f.write(bytes(t))
            for t in self.textures:
                h, w = t["rgba8"].shape[:2]
                f.write(struct.pack("<7i", w, h, t["srgb"], t["wrapS"], t["wrapT"], t["magFilter"], t["minFilter"]))
                f.write(np.ascontiguousarray(t["rgba8"], np.uint8).tobytes())
            for l in self.lights:
                f.write(bytes(l))
            if env_rgb is None:
                f.write(struct.pack("<2I", 0, 0))
            else:
                e = np.ascontiguousarray(env_rgb, "<f4")
                f.write(struct.pack("<2I", e.shape[1], e.shape[0]))
                f.write(e.tobytes())
            # optional trailing section: the EXT_mesh_opacity_micromap arrays (SceneOmm's input)
            if self.prim_omms:
                f.write(b"OMM1")
                f.write(struct.pack("<2I", len(self.micromaps), len(self.prim_omms)))
                for m in self.micromaps:
                    data = np.ascontiguousarray(m["data"], np.uint8)
                    tris = np.ascontiguousarray(m["triangles"], abi.MICROMAP_TRIANGLE_DTYPE)
                    f.write(struct.pack("<QI", data.size, tris.size))
                    f.write(data.tobytes())
                    f.write(tris.tobytes())
                for po in self.prim_omms:
                    idx = None if po.get("indices") is None else np.ascontiguousarray(po["indices"], "<i4")
                    f.write(struct.pack("<4I", po["renderPrimID"], po["micromap"], po.get("baseTriangle", 0), 0 if idx is None else idx.size))
                    if idx is not None:
                        f.write(idx.tobytes())


def _glm(m):
    """4x4 (row, col) math matrix -> glm column-major float32[16]."""
    return np.ascontiguousarray(np.asarray(m, np.float64).T.reshape(16), np.float32)


def default_material():
    """GltfShadeMaterial member defaults (gltf_scene_io.h.slang:147-310) overlaid with the glTF /
    KHR extension defaults populateShaderMaterial writes (gltf_material_cache.cpp:103-233;
    tinygltf_utils.hpp:50-248)."""
    m = abi.ShadeMaterial()
    m.pbrBaseColorFactor[:] = [1, 1, 1, 1]
    m.normalTextureScale = 1.0
    m.pbrRoughnessFactor = 1.0
    m.pbrMetallicFactor = 1.0
    m.alphaCutoff = 0.5
    m.occlusionStrength = 1.0
    m.attenuationColor[:] = [1, 1, 1]
    m.ior = 1.5
    m.attenuationDistance = float(np.finfo(np.float32).max)
    m.specularColorFactor[:] = [1, 1, 1]
    m.specularFactor = 1.0
    m.iridescenceThicknessMinimum = 100.0
    m.iridescenceThicknessMaximum = 400.0
    m.iridescenceIor = 1.3
    m.pbrDiffuseFactor[:] = [1, 1, 1, 1]
    m.pbrSpecularFactor[:] = [1, 1, 1]
    m.pbrGlossinessFactor = 1.0
    m.diffuseTransmissionColor[:] = [1, 1, 1]
    return m


# ------------------------------------------------------------------------------------------------
# glTF parsing
# ------------------------------------------------------------------------------------------------
class _Gltf:
    def __init__(self, path):
        self.dir = os.path.dirname(os.path.abspath(path))
        raw = open(path, "rb").read()
        self.bin_chunk = None
        if raw[:4] == b"glTF":
            _, _, total = struct.unpack("<4sII", raw[:12])
            off = 12
            self.json = None
            while off < total:
                clen, ctype = struct.unpack("<II", raw[off:off + 8])
                data = raw[off + 8: off + 8 + clen]
                if ctype == 0x4E4F534A:
                    self.json = json.loads(data.decode("utf-8"))
                elif ctype == 0x004E4942:
                    self.bin_chunk = data
                off += 8 + clen
        else:
            self.json = json.loads(raw.decode("utf-8"))
        self._buffers = {}

    def buffer(self, i):
        if i not in self._buffers:
            b = self.json["buffers"][i]
            uri = b.get("uri")
            if uri is None:
                data = self.bin_chunk
            elif uri.startswith("data:"):
                data = base64.b64decode(uri.split(",", 1)[1])
            else:
                data = open(os.path.join(self.dir, uri), "rb").read()
            self._buffers[i] = data
        return self._buffers[i]

    def view_bytes(self, idx):
        """raw bytes of a bufferView (None when the index or its buffer is out of range)"""
        views = self.json.get("bufferViews", [])
        if not (isinstance(idx, int) and 0 <= idx < len(views)):
            return None
        bv = views[idx]
        if not (0 <= bv.get("buffer", -1) < len(self.json.get("buffers", []))):
            return None
        buf = self.buffer(bv["buffer"])
        off = bv.get("byteOffset", 0)
        return bytes(buf[off: off + bv["byteLength"]]), bv.get("byteStride", 0)

    def accessor(self, idx, normalize=True):
        """Decode an accessor to float32 (normalized ints -> [0,1]/[-1,1]) or its integer type.
        reference: tinygltf::utils::getAccessorData / copyAccessorData (tinygltf_utils.hpp:756-)."""
        a = self.json["accessors"][idx]
        dt = np.dtype(_COMP[a["componentType"]])
        nc = _NCOMP[a["type"]]
        count = a["count"]
        if "bufferView" in a:
            bv = self.json["bufferViews"][a["bufferView"]]
            buf = self.buffer(bv["buffer"])
            start = bv.get("byteOffset", 0) + a.get("byteOffset", 0)
            stride = bv.get("byteStride", 0) or dt.itemsize * nc
            if stride == dt.itemsize * nc:
                arr = np.frombuffer(buf, dt, count * nc, start).reshape(count, nc)
            else:
                arr = np.ndarray((count, nc), dt, buf, start, (stride, dt.itemsize))
            arr = np.array(arr)
        else:
            arr = np.zeros((count, nc), dt)
        if "sparse" in a:
            sp = a["sparse"]
            ibv = self.json["bufferViews"][sp["indices"]["bufferView"]]
            idt = np.dtype(_COMP[sp["indices"]["componentType"]])
            ii = np.frombuffer(self.buffer(ibv["buffer"]), idt, sp["count"],
                               ibv.get("byteOffset", 0) + sp["indices"].get("byteOffset", 0))
            vbv = self.json["bufferViews"][sp["values"]["bufferView"]]
            vv = np.frombuffer(self.buffer(vbv["buffer"]), dt, sp["count"] * nc,
                               vbv.get("byteOffset", 0) + sp["values"].get("byteOffset", 0)).reshape(-1, nc)
            arr[ii] = vv
        if dt == np.float32 or not normalize:
            return arr
        if a.get("normalized", False):
            if dt == np.uint8:
                return (arr / 255.0).astype(np.float32)
            if dt == np.uint16:
                return (arr / 65535.0).astype(np.float32)
            if dt == np.int8:
                return np.maximum(arr / 127.0, -1.0).astype(np.float32)
            if dt == np.int16:
                return np.maximum(arr / 32767.0, -1.0).astype(np.float32)
        return arr.astype(np.float32)


def _node_matrix(node):
    """tinygltf::utils::getNodeMatrix (tinygltf_utils.cpp:641-654): matrix, else T*R*S."""
    if "matrix" in node:
        return np.asarray(node["matrix"], np.float64).reshape(4, 4).T
    t = np.asarray(node.get("translation", [0, 0, 0]), np.float64)
    q = np.asarray(node.get("rotation", [0, 0, 0, 1]), np.float64)
    s = np.asarray(node.get("scale", [1, 1, 1]), np.float64)
    return _trs(t, q, s)


def _trs(t, q, s):
    x, y, z, w = q
    r = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                  [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                  [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
    m = np.eye(4)
    m[:3, :3] = r * s[None, :]
    m[:3, 3] = t
    return m


def _pack_unorm4x8(c):
    """glm::packUnorm4x8: round(clamp(c,0,1)*255), x in the low byte."""
    q = np.round(np.clip(c, 0.0, 1.0) * 255.0).astype(np.uint32)
    return (q[:, 0] | (q[:, 1] << 8) | (q[:, 2] << 16) | (q[:, 3] << 24)).astype(np.uint32)


def _tex_transform(tinfo):
    """KHR_texture_transform -> float3x2 exactly as getTextureInfoImpl builds it
    (gltf_material_cache.cpp:84-88 from tinygltf_utils.hpp:66-85)."""
    ext = tinfo.get("extensions", {}).get("KHR_texture_transform")
    if not ext:
        return (1, 0, 0, 1, 0, 0)
    ox, oy = ext.get("offset", [0, 0])
    rot = ext.get("rotation", 0.0)
    sx, sy = ext.get("scale", [1, 1])
    c, s = math.cos(rot), math.sin(rot)
    return (sx * c, -sy * s, sx * s, sy * c, ox, oy)


def make_light(gll, world):
    """glTF KHR_lights_punctual light (JSON dict) placed by its node's world matrix (math 4x4) -> GltfLight
    (gltf_scene_vk.cpp:1354-1394)"""
    L = abi.Light()
    L.position[:] = world[:3, 3].tolist()
    L.direction[:] = (-world[:3, 2]).tolist()
    spot = gll.get("spot", {})
    L.innerAngle = spot.get("innerConeAngle", 0.0)
    L.outerAngle = spot.get("outerConeAngle", math.pi / 4)
    L.color[:] = gll.get("color", [1, 1, 1])
    L.intensity = gll.get("intensity", 1.0)
    L.type = {"point": 3, "spot": 2}.get(gll.get("type"), 1)
    ex = gll.get("extras")
    L.radius = float(ex.get("radius", 0.0)) if isinstance(ex, dict) else 0.0
    if L.type == 1:
        L.angularSizeOrInvRange = 2.0 * math.atan(L.radius / 149597870.0)
    else:
        rng = gll.get("range", 0.0)
        L.angularSizeOrInvRange = 1.0 / rng if rng > 0 else 0.0
    return L


def node_visible(node):
    """KHR_node_visibility flag of one glTF node (JSON dict), its own, not inherited"""
    return bool(node.get("extensions", {}).get("KHR_node_visibility", {}).get("visible", True))


def populate_shade_material(sm, add_texture_info):
    """tinygltf::Material (here: the glTF JSON dict) -> GltfShadeMaterial, field by field like
    MaterialCache::populateShaderMaterial (src/gltf_material_cache.cpp:63-233).  `add_texture_info(index, texCoord,
    uvTransform)` appends a GltfTextureInfo and returns its slot (> 0; slot 0 is the "no texture" sentinel)."""
    def handle(mat, slot, tinfo):
        if tinfo is not None and tinfo.get("index", -1) != -1:
            setattr(mat, slot, add_texture_info(tinfo["index"], tinfo.get("texCoord", 0), _tex_transform(tinfo)))

    m = default_material()
    am = sm.get("alphaMode", "OPAQUE")
    m.alphaMode = 0 if am == "OPAQUE" else (1 if am == "MASK" else 2)
    m.alphaCutoff = sm.get("alphaCutoff", 0.5)
    m.doubleSided = 1 if sm.get("doubleSided", False) else 0
    pbr = sm.get("pbrMetallicRoughness", {})
    m.pbrBaseColorFactor[:] = pbr.get("baseColorFactor", [1, 1, 1, 1])
    m.pbrMetallicFactor = pbr.get("metallicFactor", 1.0)
    m.pbrRoughnessFactor = pbr.get("roughnessFactor", 1.0)
    m.normalTextureScale = (sm.get("normalTexture") or {}).get("scale", 1.0)
    m.occlusionStrength = (sm.get("occlusionTexture") or {}).get("strength", 1.0)
    m.emissiveFactor[:] = sm.get("emissiveFactor", [0, 0, 0])
    handle(m, "emissiveTexture", sm.get("emissiveTexture"))
    handle(m, "normalTexture", sm.get("normalTexture"))
    handle(m, "pbrBaseColorTexture", pbr.get("baseColorTexture"))
    handle(m, "pbrMetallicRoughnessTexture", pbr.get("metallicRoughnessTexture"))
    handle(m, "occlusionTexture", sm.get("occlusionTexture"))
    ex = sm.get("extensions", {})
    e = ex.get("KHR_materials_transmission", {})
    m.transmissionFactor = e.get("transmissionFactor", 0.0)
    handle(m, "transmissionTexture", e.get("transmissionTexture"))
    m.ior = ex.get("KHR_materials_ior", {}).get("ior", 1.5)
    e = ex.get("KHR_materials_volume", {})
    m.attenuationColor[:] = e.get("attenuationColor", [1, 1, 1])
    m.thicknessFactor = e.get("thicknessFactor", 0.0)
    m.attenuationDistance = min(e.get("attenuationDistance", float(np.finfo(np.float32).max)),
                                float(np.finfo(np.float32).max))
    handle(m, "thicknessTexture", e.get("thicknessTexture"))
    e = ex.get("KHR_materials_clearcoat", {})
    m.clearcoatFactor = e.get("clearcoatFactor", 0.0)
    m.clearcoatRoughness = e.get("clearcoatRoughnessFactor", 0.0)
    handle(m, "clearcoatRoughnessTexture", e.get("clearcoatRoughnessTexture"))
    handle(m, "clearcoatTexture", e.get("clearcoatTexture"))
    handle(m, "clearcoatNormalTexture", e.get("clearcoatNormalTexture"))
    e = ex.get("KHR_materials_specular", {})
    m.specularFactor = e.get("specularFactor", 1.0)
    m.specularColorFactor[:] = e.get("specularColorFactor", [1, 1, 1])
    handle(m, "specularTexture", e.get("specularTexture"))
    handle(m, "specularColorTexture", e.get("specularColorTexture"))
    strength = ex.get("KHR_materials_emissive_strength", {}).get("emissiveStrength", 1.0)
    for k in range(3):
        m.emissiveFactor[k] = m.emissiveFactor[k] * strength
    m.unlit = 1 if "KHR_materials_unlit" in ex else 0
    e = ex.get("KHR_materials_iridescence", {})
    m.iridescenceFactor = e.get("iridescenceFactor", 0.0)
    m.iridescenceIor = e.get("iridescenceIor", 1.3)
    m.iridescenceThicknessMinimum = e.get("iridescenceThicknessMinimum", 100.0)
    m.iridescenceThicknessMaximum = e.get("iridescenceThicknessMaximum", 400.0)
    handle(m, "iridescenceTexture", e.get("iridescenceTexture"))
    handle(m, "iridescenceThicknessTexture", e.get("iridescenceThicknessTexture"))
    e = ex.get("KHR_materials_anisotropy", {})
    rot = e.get("anisotropyRotation", 0.0)
    m.anisotropyRotation[:] = [math.sin(rot), math.cos(rot)]
    m.anisotropyStrength = e.get("anisotropyStrength", 0.0)
    handle(m, "anisotropyTexture", e.get("anisotropyTexture"))
    e = ex.get("KHR_materials_sheen", {})
    m.sheenColorFactor[:] = e.get("sheenColorFactor", [0, 0, 0])
    m.sheenRoughnessFactor = e.get("sheenRoughnessFactor", 0.0)
    handle(m, "sheenColorTexture", e.get("sheenColorTexture"))
    handle(m, "sheenRoughnessTexture", e.get("sheenRoughnessTexture"))
    m.dispersion = ex.get("KHR_materials_dispersion", {}).get("dispersion", 0.0)
    if "KHR_materials_pbrSpecularGlossiness" in ex:
        e = ex["KHR_materials_pbrSpecularGlossiness"]
        m.pbrModel = 1
        m.pbrDiffuseFactor[:] = e.get("diffuseFactor", [1, 1, 1, 1])
        m.pbrSpecularFactor[:] = e.get("specularFactor", [1, 1, 1])
        m.pbrGlossinessFactor = e.get("glossinessFactor", 1.0)
        handle(m, "pbrDiffuseTexture", e.get("diffuseTexture"))
        handle(m, "pbrSpecularGlossinessTexture", e.get("specularGlossinessTexture"))
    e = ex.get("KHR_materials_diffuse_transmission", {})
    m.diffuseTransmissionFactor = e.get("diffuseTransmissionFactor", 0.0)
    m.diffuseTransmissionColor[:] = e.get("diffuseTransmissionColorFactor", [1, 1, 1])
    handle(m, "diffuseTransmissionTexture", e.get("diffuseTransmissionTexture"))
    handle(m, "diffuseTransmissionColorTexture", e.get("diffuseTransmissionColorTexture"))
    e = ex.get("KHR_materials_retroreflection", {})
    m.retroreflectionFactor = e.get("retroreflectionFactor", 0.0)
    handle(m, "retroreflectionTexture", e.get("retroreflectionTexture"))
    e = ex.get("KHR_materials_volume_scatter", {})
    m.multiscatterColorFactor[:] = e.get("multiscatterColorFactor", e.get("multiscatterColor", [0, 0, 0]))
    m.scatterAnisotropy = e.get("scatterAnisotropy", 0.0)
    return m


class MaterialCache:
    """Host mirror of nvvkgltf::MaterialCache (src/gltf_material_cache.{hpp,cpp}): the GltfShadeMaterial[] and
    GltfTextureInfo[] arrays the path tracer consumes, rebuilt from the glTF materials, with in-place updates that report
    whether the set of bound textures (the array topology) changed.  Pinned by the reference's own expectations
    (tests/test_material_cache.cpp:24-176) in tests/test_material_cache.py."""

    class UpdateResult:
        def __init__(self, topology_changed=False, span=None):
            self.topologyChanged = topology_changed
            self.span = span  # (first, count) of the materials rewritten, None = nothing

        def hasAny(self):
            return self.span is not None

    def __init__(self):
        self.clear()

    def clear(self):
        self._materials = []
        self._texture_infos = []
        self._sources = []

    def _add_ti(self, index, texcoord, uv_transform):
        ti = abi.TextureInfo()
        ti.index = index
        ti.texCoord = min(texcoord, 1)  # the shaders know TEXCOORD_0 and TEXCOORD_1 only
        ti.uvTransform[:] = list(uv_transform)
        self._texture_infos.append(ti)
        return len(self._texture_infos) - 1

    def buildFromMaterials(self, materials):
        self.clear()
        sentinel = abi.TextureInfo()
        sentinel.index = -1
        sentinel.uvTransform[:] = [1, 0, 0, 1, 0, 0]
        self._texture_infos = [sentinel]  # slot 0: "no texture"
        for sm in materials:
            self._materials.append(populate_shade_material(sm, self._add_ti))
            self._sources.append(sm)

    @staticmethod
    def _bound_slots(m):
        return tuple(getattr(m, n) > 0 for n in abi.MATERIAL_TEXTURE_SLOTS)

    def updateMaterial(self, index, sm):
        if index < 0 or index >= len(self._materials):
            return MaterialCache.UpdateResult(False, None)
        before = self._bound_slots(self._materials[index])
        scratch = []

        def probe(i, tc, xf):
            scratch.append((i, tc, xf))
            return len(scratch)
        after = self._bound_slots(populate_shade_material(sm, probe))
        if after != before:
            # a texture was added or removed: every slot index behind it moves -> rebuild (the reference re-creates the arrays)
            srcs = list(self._sources)
            srcs[index] = sm
            self.buildFromMaterials(srcs)
            return MaterialCache.UpdateResult(True, (0, len(self._materials)))
        # same topology: rewrite the material in place; its texture infos keep their slots and are refreshed
        old = self._materials[index]
        rec = []

        def record(i, tc, xf):
            rec.append((i, tc, xf))
            return len(rec)
        new = populate_shade_material(sm, record)  # texture slots hold the visit number 1..n
        for n in abi.MATERIAL_TEXTURE_SLOTS:
            k = getattr(new, n)
            if k > 0:
                slot = getattr(old, n)
                i, tc, xf = rec[k - 1]
                ti = self._texture_infos[slot]
                ti.index, ti.texCoord = i, min(tc, 1)
                ti.uvTransform[:] = list(xf)
                setattr(new, n, slot)
        self._materials[index] = new
        self._sources[index] = sm
        return MaterialCache.UpdateResult(False, (index, 1))

    def getShadeMaterials(self):
        return self._materials

    def getTextureInfos(self):
        return self._texture_infos


def load_gltf(path):
    g = _Gltf(path)
    j = g.json
    scn = Scene()

    # ---- textures / images (SceneVk::createTextureImages) ----
    images = j.get("images", [])
    srgb_images = set()

    def tex_image(tex_id):
        t = j["textures"][tex_id]
        for e in ("KHR_texture_basisu", "EXT_texture_webp", "MSFT_texture_dds", "EXT_texture_avif"):
            if e in t.get("extensions", {}):
                return t["extensions"][e]["source"]
        return t.get("source", -1)

    def mark_srgb(tinfo):
        if tinfo and tinfo.get("index", -1) > -1:
            srgb_images.add(tex_image(tinfo["index"]))

    for m in j.get("materials", []):
        mark_srgb(m.get("pbrMetallicRoughness", {}).get("baseColorTexture"))
        mark_srgb(m.get("emissiveTexture"))
        ex = m.get("extensions", {})
        mark_srgb(ex.get("KHR_materials_specular", {}).get("specularColorTexture"))
        mark_srgb(ex.get("KHR_materials_sheen", {}).get("sheenColorTexture"))
        mark_srgb(ex.get("KHR_materials_pbrSpecularGlossiness", {}).get("diffuseTexture"))
        mark_srgb(ex.get("KHR_materials_pbrSpecularGlossiness", {}).get("specularGlossinessTexture"))
    for t in j.get("textures", []):
        ex = t.get("extras")
        if isinstance(ex, dict) and float(ex.get("gamma", 0)) > 1.0:
            srgb_images.add(tex_image(j["textures"].index(t)))

    decoded = {}

    def decode_image(i):
        if i in decoded:
            return decoded[i]
        from PIL import Image
        try:
            im = images[i]
            if "uri" in im:
                if im["uri"].startswith("data:"):
                    data = base64.b64decode(im["uri"].split(",", 1)[1])
                else:
                    data = open(os.path.join(g.dir, im["uri"]), "rb").read()
            else:
                bv = j["bufferViews"][im["bufferView"]]
                data = g.buffer(bv["buffer"])[bv.get("byteOffset", 0): bv.get("byteOffset", 0) + bv["byteLength"]]
            arr = np.asarray(Image.open(io.BytesIO(data)).convert("RGBA"), np.uint8)
        except Exception:
            arr = np.array([[[255, 0, 255, 255]]], np.uint8)  # magenta default (gltf_scene_vk.cpp:1054-1060)
        decoded[i] = np.ascontiguousarray(arr)
        return decoded[i]

    for ti, t in enumerate(j.get("textures", [])):
        src = tex_image(ti)
        smp = j["samplers"][t["sampler"]] if t.get("sampler", -1) > -1 else {}
        rgba = decode_image(src) if src > -1 else np.array([[[255, 255, 255, 255]]], np.uint8)
        scn.add_texture(rgba, srgb=(src in srgb_images), wrapS=smp.get("wrapS", 10497), wrapT=smp.get("wrapT", 10497),
                        magFilter=smp.get("magFilter", -1), minFilter=smp.get("minFilter", -1))

    # ---- materials (MaterialCache::buildFromMaterials) ----
    src_mats = j.get("materials", []) or [{}]
    for sm in src_mats:
        scn.materials.append(populate_shade_material(sm, scn.add_texture_info))

    # ---- unique primitives (Scene::buildPrimitiveKeyMap) ----
    prim_map = {}

    def prim_key(p):
        key = " ".join(f"{k}:{v}" for k, v in sorted(p["attributes"].items())) + f" indices:{p.get('indices', -1)}"
        for t in p.get("targets", []):
            key += " target:" + ",".join(f"{k}:{v}" for k, v in sorted(t.items()))
        return key

    for mesh_id, mesh in enumerate(j.get("meshes", [])):
        for p in mesh["primitives"]:
            if p.get("mode", 4) != 4:
                continue
            key = prim_key(p)
            if key in prim_map:
                continue
            at = p["attributes"]
            pos = g.accessor(at["POSITION"])
            if "indices" in p:
                idx = g.accessor(p["indices"], normalize=False).astype(np.uint32).reshape(-1)
            else:
                idx = np.arange(len(pos), dtype=np.uint32)
            idx = idx[: (len(idx) // 3) * 3].reshape(-1, 3)
            colors = None
            if "COLOR_0" in at:
                c = g.accessor(at["COLOR_0"])
                if c.shape[1] == 3:
                    c = np.concatenate([c, np.ones((len(c), 1), np.float32)], 1)
                colors = _pack_unorm4x8(c)
            prim_map[key] = scn.add_primitive(
                pos, idx,
                normals=g.accessor(at["NORMAL"]) if "NORMAL" in at else None,
                uv0=g.accessor(at["TEXCOORD_0"]) if "TEXCOORD_0" in at else None,
                uv1=g.accessor(at["TEXCOORD_1"]) if "TEXCOORD_1" in at else None,
                tangents=g.accessor(at["TANGENT"]) if "TANGENT" in at else None,
                colors=colors)
            pid = prim_map[key]
            # morph targets (parseMorphTargets, gltf_scene_animation.cpp:150-262) and skin attributes (parseSkinTasks, :270-316)
            targets = p.get("targets", [])
            if targets and all("POSITION" in t for t in targets):
                def stack(name):
                    if not any(name in t for t in targets):
                        return None
                    return np.stack([g.accessor(t[name]).astype(np.float32)[:, :3] if name in t else np.zeros((len(pos), 3), np.float32) for t in targets])
                scn.morph_prims[pid] = dict(mesh=mesh_id, position_deltas=stack("POSITION"), normal_deltas=stack("NORMAL"), tangent_deltas=stack("TANGENT"))
            if "JOINTS_0" in at and "WEIGHTS_0" in at:
                scn.skin_prims[pid] = dict(joints=g.accessor(at["JOINTS_0"], normalize=False).astype(np.int32).reshape(-1, 4),
                                           weights=g.accessor(at["WEIGHTS_0"]).astype(np.float32).reshape(-1, 4))

    # ---- EXT_mesh_opacity_micromap (SceneOmm::create, src/gltf_scene_omm.cpp:140-391): root micromaps[] + per-primitive linkage.
    # Malformed entries are skipped with the reference's rules (missing required field, bad bufferView, misaligned usage arrays,
    # negative base triangle, bad indices accessor); rendering then falls back to the regular alpha path for those primitives.
    omm_root = j.get("extensions", {}).get("EXT_mesh_opacity_micromap")
    if isinstance(omm_root, dict) and isinstance(omm_root.get("micromaps"), list):
        slot_of = {}
        for i, mm in enumerate(omm_root["micromaps"]):
            if not all(k in mm for k in ("data", "triangles", "usageCounts", "usageLevels", "usageFormats")):
                continue
            uc, ul, uf = mm["usageCounts"], mm["usageLevels"], mm["usageFormats"]
            if not (isinstance(uc, list) and isinstance(ul, list) and isinstance(uf, list) and len(uc) == len(ul) == len(uf)):
                continue
            dv, tv = g.view_bytes(mm["data"]), g.view_bytes(mm["triangles"])
            if dv is None or tv is None:
                continue
            stride = tv[1] or 8
            raw = np.frombuffer(tv[0], np.uint8)
            n = len(raw) // stride if stride > 8 else len(raw) // 8
            if stride > 8:
                raw = np.ascontiguousarray(raw[: n * stride].reshape(n, stride)[:, :8]).reshape(-1)
            tris = np.frombuffer(raw[: n * 8].tobytes(), abi.MICROMAP_TRIANGLE_DTYPE)
            slot_of[i] = len(scn.micromaps)
            scn.micromaps.append(dict(data=np.frombuffer(dv[0], np.uint8).copy(), triangles=tris.copy()))
        linked = set()
        for mesh in j.get("meshes", []):
            for p in mesh["primitives"]:
                ext = p.get("extensions", {}).get("EXT_mesh_opacity_micromap")
                if p.get("mode", 4) != 4 or not isinstance(ext, dict) or "micromap" not in ext:
                    continue
                pid = prim_map[prim_key(p)]
                if ext["micromap"] not in slot_of or pid in linked:
                    continue
                base = ext.get("micromapBaseTriangle", 0)
                if base < 0:
                    continue
                idx = None
                if "micromapIndices" in ext:
                    ai = ext["micromapIndices"]
                    if not (isinstance(ai, int) and 0 <= ai < len(j.get("accessors", []))):
                        continue
                    raw_idx = np.ascontiguousarray(g.accessor(ai, normalize=False).reshape(-1))
                    # the index buffer is typed like a VkIndexType: the special indices are -1..-4 in the accessor's own width
                    idx = raw_idx.view(np.dtype("i%d" % raw_idx.dtype.itemsize)).astype(np.int32)
                linked.add(pid)
                scn.prim_omms.append(dict(renderPrimID=pid, micromap=slot_of[ext["micromap"]], baseTriangle=int(base), indices=idx))

    # ---- scene graph (Scene::parseScene) ----
    nodes = j.get("nodes", [])
    gl_lights = j.get("extensions", {}).get("KHR_lights_punctual", {}).get("lights", [])
    scene_id = j.get("scene", 0)
    cam_found = []

    parents = np.full(len(nodes), -1, np.int32)
    for nid, node in enumerate(nodes):
        for c in node.get("children", []):
            parents[c] = nid
    skins = []
    for sk in j.get("skins", []):
        ibm = None
        if "inverseBindMatrices" in sk:
            ibm = g.accessor(sk["inverseBindMatrices"]).astype(np.float64).reshape(-1, 4, 4).transpose(0, 2, 1)   # glm column-major -> (row, col)
        skins.append(dict(joints=list(sk.get("joints", [])), ibm=ibm))
    # animations as AnimationSystem::parseAnimations caches them: per sampler the key times, the decoded outputs with their accessor
    # type and the interpolation; per channel its target, and for a "pointer" channel the KHR_animation_pointer string (empty
    # without the extension: gltf_scene_animation.cpp:182-188)
    animations = []
    for an in j.get("animations", []):
        samplers = []
        for sm in an.get("samplers", []):
            samplers.append(dict(inputs=g.accessor(sm["input"]).astype(np.float32).reshape(-1), outputs=g.accessor(sm["output"]).astype(np.float32),
                                 type=j["accessors"][sm["output"]]["type"], interpolation=sm.get("interpolation", "LINEAR")))
        channels = []
        for ch in an.get("channels", []):
            tgt = ch.get("target", {})
            pointer = tgt.get("extensions", {}).get("KHR_animation_pointer", {}).get("pointer", "") if tgt.get("path") == "pointer" else ""
            channels.append(dict(node=tgt.get("node", -1), path=tgt.get("path", ""), sampler=ch["sampler"], pointer=pointer))
        animations.append(dict(name=an.get("name", ""), samplers=samplers, channels=channels))
    scn.graph = dict(parents=parents, locals=np.asarray([_node_matrix(n) for n in nodes], np.float64).reshape(-1, 4, 4), render_nodes=[], skins=skins,
                     mesh_weights={m: np.asarray(mesh.get("weights", []), np.float32) for m, mesh in enumerate(j.get("meshes", []))},
                     trs=[dict(matrix=n.get("matrix"), translation=n.get("translation", [0, 0, 0]), rotation=n.get("rotation", [0, 0, 0, 1]),
                               scale=n.get("scale", [1, 1, 1]), mesh=n.get("mesh", -1)) for n in nodes], animations=animations)

    def visit(nid, parent):
        node = nodes[nid]
        world = parent @ _node_matrix(node)
        if "camera" in node and not cam_found:
            cam_found.append((nid, world))
        li = node.get("extensions", {}).get("KHR_lights_punctual", {}).get("light", -1)
        if 0 <= li < len(gl_lights):
            scn.lights.append(make_light(gl_lights[li], world))
            scn.light_sources.append((li, world))
        if node.get("mesh", -1) > -1:
            inst = node.get("extensions", {}).get("EXT_mesh_gpu_instancing")
            locals_ = [np.eye(4)]
            if inst:
                at = inst["attributes"]
                T = g.accessor(at["TRANSLATION"]) if "TRANSLATION" in at else None
                R = g.accessor(at["ROTATION"]) if "ROTATION" in at else None
                S = g.accessor(at["SCALE"]) if "SCALE" in at else None
                n = max(len(x) for x in (T, R, S) if x is not None)
                locals_ = [_trs(T[i] if T is not None and i < len(T) else np.zeros(3),
                                R[i] if R is not None and i < len(R) else np.array([0, 0, 0, 1.0]),
                                S[i] if S is not None and i < len(S) else np.ones(3)) for i in range(n)]
            for p in j["meshes"][node["mesh"]]["primitives"]:
                if p.get("mode", 4) != 4:
                    continue
                variant_materials = {v: mp["material"] for mp in p.get("extensions", {}).get("KHR_materials_variants", {}).get("mappings", [])
                                     for v in mp.get("variants", []) if "material" in mp}
                for lm in locals_:
                    scn.add_node(prim_map[prim_key(p)], p.get("material", -1), world @ lm)
                    scn.render_nodes[-1].update(defaultMaterial=p.get("material", -1), variantMaterials=variant_materials)
                    scn.graph["render_nodes"].append((nid, node.get("skin", -1), np.asarray(lm, np.float64)))   # RenderNode::refNodeID / skinID
        for c in node.get("children", []):
            visit(c, world)

    for root in j.get("scenes", [{"nodes": list(range(len(nodes)))}])[scene_id]["nodes"]:
        visit(root, np.eye(4))
    scn.variants = [v.get("name", "") for v in j.get("extensions", {}).get("KHR_materials_variants", {}).get("variants", [])]
    scn.node_visible = [node_visible(n) for n in nodes]
    scn._apply_visibility()
    scn.gltf = j

    # ---- camera (Scene::handleCameraTraversal) ----
    if cam_found:
        nid, world = cam_found[0]
        gc = j["cameras"][nodes[nid]["camera"]]
        cam = Camera()
        lo, hi = scn.bounds() if scn.render_nodes else (np.full(3, -1.0), np.full(3, 1.0))
        center = (lo + hi) * 0.5
        radius = float(np.linalg.norm(hi - lo) * 0.5)
        if gc["type"] == "perspective":
            pp = gc["perspective"]
            cam.yfov, cam.znear, cam.zfar = pp["yfov"], pp["znear"], pp.get("zfar", 0.0)
        else:
            cam.type = "orthographic"
            oo = gc["orthographic"]
            cam.xmag, cam.ymag, cam.znear, cam.zfar = oo["xmag"], oo["ymag"], oo["znear"], oo["zfar"]
        if cam.zfar <= cam.znear:
            cam.zfar = max(cam.znear * 2.0, 4.0 * radius)
        # extractCameraVectors: eye = translation, forward = -Z, center at the scene-centre distance
        eye = world[:3, 3]
        fwd = -world[:3, 2] / max(np.linalg.norm(world[:3, 2]), 1e-20)
        dist = float(np.linalg.norm(center - eye))
        cam.eye, cam.center, cam.up = eye.astype(np.float32), (eye + fwd * dist).astype(np.float32), \
            (world[:3, 1] / max(np.linalg.norm(world[:3, 1]), 1e-20)).astype(np.float32)
        ex = nodes[nid].get("extras")
        if isinstance(ex, dict):
            if "camera::eye" in ex:
                cam.eye = np.asarray(ex["camera::eye"], np.float32)
            if "camera::center" in ex:
                cam.center = np.asarray(ex["camera::center"], np.float32)
            if "camera::up" in ex:
                cam.up = np.asarray(ex["camera::up"], np.float32)
        scn.camera = cam
    return scn
