// refit.cuh — refit of the compressed wide BVH after the render nodes' transforms changed (device code).
//
// Reference: the TLAS update / BLAS refit path of SceneRtx (src/gltf_scene_rtx.cpp:416-503: updateTopLevelAS with
// VK_BUILD_ACCELERATION_STRUCTURE_MODE_UPDATE_KHR when instance matrices move, :551-565 updateBottomLevelAS) -- the driver refits
// its hardware BVH; here the flattened world-space tree is refitted:
//   1. k_refit_tris   every triangle record is recomputed from its primitive's object-space vertices and its node's NEW
//                     objectToWorld (the same arithmetic, operation by operation, as the host flatten in b200pt_set_scene, so a
//                     refitted tree answers every ray exactly like a freshly built one),
//   2. k_refit_level  bottom-up, one launch per tree level (nodes of a level are contiguous: the builders emit breadth first):
//                     a node's child boxes are re-read (leaf children from their triangles, inner children from the boxes the level
//                     below stored), its own box is their union, and the node is re-quantised in a new frame.  Topology (child
//                     slots, axis map, triangle order) is kept.
#pragma once
#include "bvh.h"
#include "device_scene.cuh"

namespace pt {

// box of the triangle the walks intersect (v0, v0 + e1, v0 + e2: T is its 12-float record), padded like the host builder's leaf
// boxes (bvh.cpp) because the vertex sums are rounded: both builders and the refit bound a triangle the same way
PT_D void triangleBox(const float* T, float lo[3], float hi[3])
{
  for(int a = 0; a < 3; a++)
  {
    const float v0 = T[a], v1 = T[a] + T[4 + a], v2 = T[a] + T[8 + a];
    const float l = fminf(v0, fminf(v1, v2)), h = fmaxf(v0, fmaxf(v1, v2));
    const float pad = fmaxf(fabsf(l), fabsf(h)) * 4e-7f + 1e-30f;
    lo[a] = l - pad;
    hi[a] = h + pad;
  }
}

// conservative quantisation of one node, the host builder's arithmetic (bvh.cpp "quantisation frame")
PT_D void quantiseNode(float* N, const float lo[3], const float hi[3], const float clo[8][3], const float chi[8][3], uint32_t present)
{
  uint32_t eb[3];
  double   scale[3];
  for(int a = 0; a < 3; a++)
  {
    const double ext = (double)hi[a] - (double)lo[a];
    int          e = (ext > 0.0) ? (int)ceil(log2(ext / 255.0)) : -126;
    while(ldexp(255.0, e) < ext)
      e++;
    e = e < -126 ? -126 : (e > 127 ? 127 : e);
    eb[a] = (uint32_t)(e + 127);
    scale[a] = ldexp(1.0, e);
  }
  uint32_t q[3][4] = {{0, 0, 0, 0}, {0, 0, 0, 0}, {0, 0, 0, 0}};  // per axis: lo[0..3], lo[4..7], hi[0..3], hi[4..7]
  for(int s = 0; s < 8; s++)
    for(int a = 0; a < 3; a++)
    {
      uint32_t ql = 255u, qh = 0u;  // empty slot: inverted box never hits
      if(present & (1u << s))
      {
        const double l = ((double)clo[s][a] - (double)lo[a]) / scale[a];
        const double h = ((double)chi[s][a] - (double)lo[a]) / scale[a];
        const int    il = (int)floor(l - 1e-3), ih = (int)ceil(h + 1e-3);
        ql = (uint32_t)(il < 0 ? 0 : (il > 255 ? 255 : il));
        qh = (uint32_t)(ih < 0 ? 0 : (ih > 255 ? 255 : ih));
      }
      q[a][s >> 2] |= ql << (8 * (s & 3));
      q[a][2 + (s >> 2)] |= qh << (8 * (s & 3));
    }
  const uint32_t imask = __float_as_uint(N[3]) >> 24;
  N[0] = lo[0];
  N[1] = lo[1];
  N[2] = lo[2];
  N[3] = __uint_as_float(eb[0] | (eb[1] << 8) | (eb[2] << 16) | (imask << 24));
  for(int a = 0; a < 3; a++)
    for(int k = 0; k < 4; k++)
      N[8 + a * 4 + k] = __uint_as_float(q[a][k]);
}

// one node of a level: child boxes -> own box -> re-quantised node.  nodeBox: 2 float4 per node (lo, hi).
PT_D void refitNode(uint32_t node, float* nodes, const float* tris, float4* nodeBox)
{
  float*         N = nodes + (size_t)node * 20;
  const uint32_t imask = __float_as_uint(N[3]) >> 24;
  const uint32_t childBase = __float_as_uint(N[4]) & 0x03ffffffu, triBase = __float_as_uint(N[5]);
  float          clo[8][3], chi[8][3], lo[3] = {3.0e38f, 3.0e38f, 3.0e38f}, hi[3] = {-3.0e38f, -3.0e38f, -3.0e38f};
  uint32_t       present = 0;
  for(int s = 0; s < 8; s++)
  {
    const uint32_t meta = (__float_as_uint(N[6 + (s >> 2)]) >> (8 * (s & 3))) & 0xffu;
    if(meta == 0u)
      continue;
    present |= 1u << s;
    if((meta & (meta << 1)) & 0x10u)
    {
      const uint32_t child = childBase + (uint32_t)__popc(imask & ((1u << s) - 1u));
      const float4   bl = nodeBox[child * 2], bh = nodeBox[child * 2 + 1];
      clo[s][0] = bl.x, clo[s][1] = bl.y, clo[s][2] = bl.z;
      chi[s][0] = bh.x, chi[s][1] = bh.y, chi[s][2] = bh.z;
    }
    else
    {
      const uint32_t count = (uint32_t)__popc(meta >> 5), first = triBase + (meta & 0x1fu);
      for(int a = 0; a < 3; a++)
      {
        clo[s][a] = 3.0e38f;
        chi[s][a] = -3.0e38f;
      }
      for(uint32_t k = 0; k < count; k++)
      {
        float tlo[3], thi[3];
        triangleBox(tris + (size_t)(first + k) * 12, tlo, thi);
        for(int a = 0; a < 3; a++)
        {
          clo[s][a] = fminf(clo[s][a], tlo[a]);
          chi[s][a] = fmaxf(chi[s][a], thi[a]);
        }
      }
    }
    for(int a = 0; a < 3; a++)
    {
      lo[a] = fminf(lo[a], clo[s][a]);
      hi[a] = fmaxf(hi[a], chi[s][a]);
    }
  }
  if(present == 0u)
  {
    lo[0] = lo[1] = lo[2] = hi[0] = hi[1] = hi[2] = 0.0f;  // the empty tree's single empty node
  }
  nodeBox[node * 2] = make_float4(lo[0], lo[1], lo[2], 0.0f);
  nodeBox[node * 2 + 1] = make_float4(hi[0], hi[1], hi[2], 0.0f);
  quantiseNode(N, lo, hi, clo, chi, present);
}

// world-space record of one triangle slot from its primitive's vertices and its node's current transform
// (b200pt_set_scene's flatten: v = objectToWorld * p, mirrored instances swap v1 / v2 and carry TRI_FLIPPED)
PT_D void refitTriangle(uint32_t slot, float* tris, uint2* triMeta, const b200pt_render_node* nodes, const DevPrim* prims)
{
  float*         T = tris + (size_t)slot * 12;
  const uint32_t w0 = __float_as_uint(T[3]), primTri = __float_as_uint(T[7]);
  const uint32_t rnode = w0 & 0x0fffffffu;
  uint32_t       flags = (w0 >> 28) & ~(uint32_t)TRI_FLIPPED;
  const b200pt_render_node& node = nodes[rnode];
  const DevPrim             P = prims[node.renderPrimID];
  const float*              a = node.objectToWorld;
  const float    det = a[0] * (a[5] * a[10] - a[9] * a[6]) - a[4] * (a[1] * a[10] - a[9] * a[2]) + a[8] * (a[1] * a[6] - a[5] * a[2]);
  float3         v[3];
  for(int k = 0; k < 3; k++)
  {
    const uint32_t vi = P.idx[primTri * 3 + k];
    v[k] = xfPoint(a, f3(P.pos[vi * 3], P.pos[vi * 3 + 1], P.pos[vi * 3 + 2]));
  }
  if(det < 0.0f)
  {
    const float3 t = v[1];
    v[1] = v[2];
    v[2] = t;
    flags |= TRI_FLIPPED;
  }
  const float3 e1 = v[1] - v[0], e2 = v[2] - v[0];
  T[0] = v[0].x, T[1] = v[0].y, T[2] = v[0].z;
  T[3] = __uint_as_float(rnode | (flags << 28));
  T[4] = e1.x, T[5] = e1.y, T[6] = e1.z;
  T[8] = e2.x, T[9] = e2.y, T[10] = e2.z;
  triMeta[slot].x = rnode | (flags << 28);
}

}  // namespace pt
