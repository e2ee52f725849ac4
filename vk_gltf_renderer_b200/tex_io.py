"""Packing of texture unit-test records for b200pt_texture_lookup (include/b200pt.h).

8 floats per record:
  0 texture-info slot (index into the scene's texture infos; 0 is the reserved "none" slot) |
  1 mode: 0 = getTexture (the shade path: texCoord select, uvTransform, texGrad footprint),
          1 = sampleLevel0 (the generic alpha test: texCoord select, level 0 with the magnification filter) |
  2-3 tc0.xy | 4-5 tc1.xy | 6 texGrad (0 = no gradient: level 0) | 7 unused
output (4 floats): rgba
"""
import numpy as np

GET_TEXTURE = 0
SAMPLE_LEVEL0 = 1


def records(slot, uv, *, mode=GET_TEXTURE, tc1=None, tex_grad=0.0):
    """One record per row of uv (float [n, 2], TEXCOORD_0); tc1 defaults to uv; slot, mode and tex_grad broadcast."""
    uv = np.asarray(uv, np.float32).reshape(-1, 2)
    r = np.zeros((len(uv), 8), np.float32)
    r[:, 0] = slot
    r[:, 1] = mode
    r[:, 2:4] = uv
    r[:, 4:6] = uv if tc1 is None else np.asarray(tc1, np.float32).reshape(-1, 2)
    r[:, 6] = tex_grad
    return r
