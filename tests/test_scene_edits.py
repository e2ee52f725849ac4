"""Scene edits on the host: KHR_materials_variants switches and inherited KHR_node_visibility of a loaded glTF, and the
scene description they produce (what PathTracer.update_node_materials / set_node_visibility hand to the library)."""
import base64
import json

import numpy as np
import pytest

from vk_gltf_renderer_b200 import scene

# render nodes of the asset below, in load order:
#   0, 1  node 1 (mesh 0, two EXT_mesh_gpu_instancing copies)        under node 0
#   2     node 2 (mesh 1)                                              under node 0
#   3     node 3 (mesh 1, hidden)                                      under node 2
#   4     node 4 (mesh 0, hidden root)
#   5     node 5 (mesh 1)                                              under node 4 (hidden by inheritance)
RED, BLUE = 0, 1


def _write_asset(path):
    pos = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], np.float32)
    trans = np.array([[0, 0, 0], [2, 0, 0]], np.float32)
    blob = pos.tobytes() + trans.tobytes()
    mapped = {"attributes": {"POSITION": 0}, "material": 0,
              "extensions": {"KHR_materials_variants": {"mappings": [{"material": 1, "variants": [RED]},
                                                                     {"material": 2, "variants": [BLUE]}]}}}
    plain = {"attributes": {"POSITION": 0}, "material": 0}
    hidden = {"KHR_node_visibility": {"visible": False}}
    g = {
        "asset": {"version": "2.0"},
        "extensionsUsed": ["KHR_materials_variants", "KHR_node_visibility", "EXT_mesh_gpu_instancing"],
        "extensions": {"KHR_materials_variants": {"variants": [{"name": "red"}, {"name": "blue"}]}},
        "buffers": [{"byteLength": len(blob), "uri": "data:application/octet-stream;base64," + base64.b64encode(blob).decode()}],
        "bufferViews": [{"buffer": 0, "byteOffset": 0, "byteLength": 36}, {"buffer": 0, "byteOffset": 36, "byteLength": 24}],
        "accessors": [{"bufferView": 0, "componentType": 5126, "count": 3, "type": "VEC3", "min": [0, 0, 0], "max": [1, 1, 0]},
                      {"bufferView": 1, "componentType": 5126, "count": 2, "type": "VEC3"}],
        "materials": [{"name": "base"}, {"name": "red"}, {"name": "blue"}],
        "meshes": [{"primitives": [mapped]}, {"primitives": [plain]}],
        "nodes": [{"children": [1, 2]},
                  {"mesh": 0, "extensions": {"EXT_mesh_gpu_instancing": {"attributes": {"TRANSLATION": 1}}}},
                  {"mesh": 1, "children": [3]},
                  {"mesh": 1, "extensions": hidden},
                  {"mesh": 0, "children": [5], "extensions": hidden},
                  {"mesh": 1}],
        "scenes": [{"nodes": [0, 4]}],
        "scene": 0,
    }
    path.write_text(json.dumps(g))
    return str(path)


@pytest.fixture
def scn(tmp_path):
    return scene.load_gltf(_write_asset(tmp_path / "edits.gltf"))


def ids(s):
    return [rn["materialID"] for rn in s.render_nodes]


def shown(s):
    return [rn["visible"] for rn in s.render_nodes]


def test_variant_names(scn):
    assert scn.variants == ["red", "blue"]
    assert len(scn.render_nodes) == 6


def test_set_variant_mapped_unmapped_and_instanced(scn):
    assert ids(scn) == [0, 0, 0, 0, 0, 0]
    scn.set_variant(RED)
    # both instanced copies and the hidden copy of mesh 0 switch; mesh 1 has no mapping and keeps its own material
    assert ids(scn) == [1, 1, 0, 0, 1, 0]
    scn.set_variant(BLUE)
    assert ids(scn) == [2, 2, 0, 0, 2, 0]
    scn.set_variant(None)
    assert ids(scn) == [0, 0, 0, 0, 0, 0]
    scn.set_variant(RED)
    assert ids(scn) == [1, 1, 0, 0, 1, 0]


def test_visibility_is_inherited(scn):
    # node 3 is hidden itself, node 5 below the hidden root 4
    assert shown(scn) == [True, True, True, False, False, False]
    scn.set_node_visible(4, True)
    assert shown(scn) == [True, True, True, False, True, True]
    scn.set_node_visible(2, False)   # hides render node 2; node 3 stays hidden
    assert shown(scn) == [True, True, False, False, True, True]
    scn.set_node_visible(0, False)   # a hidden root hides its whole subtree, instanced copies included
    assert shown(scn) == [False, False, False, False, True, True]
    scn.set_node_visible(5, False)   # a hidden leaf
    assert shown(scn) == [False, False, False, False, True, False]
    for n in range(6):
        scn.set_node_visible(n, True)
    assert shown(scn) == [True] * 6


def test_desc_carries_the_edits(scn):
    scn.set_variant(BLUE)
    scn.set_node_visible(0, False)
    d = scn.desc()
    assert d.numRenderNodes == 6 and d.numMaterials == 3
    assert [d.renderNodes[i].materialID for i in range(6)] == [2, 2, 0, 0, 2, 0]
    assert [d.renderNodeVisible[i] for i in range(6)] == [0, 0, 0, 0, 0, 0]
    scn.set_node_visible(4, True)
    d = scn.desc()
    assert [d.renderNodeVisible[i] for i in range(6)] == [0, 0, 0, 0, 1, 1]


def test_set_node_visible_needs_a_loaded_scene():
    with pytest.raises(ValueError):
        scene.Scene().set_node_visible(0, False)
