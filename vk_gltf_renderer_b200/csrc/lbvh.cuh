// lbvh.cuh — construction of the compressed 8-wide BVH ON THE DEVICE (SURVEY.md section 8f rank 1; replaces what SceneRtx asks
// the driver for: BLAS / TLAS builds, src/gltf_scene_rtx.cpp:173-388).
//
//   1. lbvhBounds     per triangle: box + centroid; scene centroid bounds by atomic min / max
//   2. lbvhMorton     30-bit Morton code of the centroid, made unique by the triangle's index in the low word of a 64-bit key
//   3. bitonicStep    sort of the keys (n log^2 n compare-exchange passes over global memory; the build is not on the frame path)
//   4. lbvhHierarchy  binary radix tree over the sorted keys, one thread per internal node (Karras 2012)
//   5. lbvhFit        bottom-up boxes: the second thread to reach a node continues upwards
//   6. lbvhEmit       collapse into 8-wide nodes level by level: a wide node starts from the two children of its binary node and
//                     keeps opening the child with the largest surface area until it has 8 (subtrees of <= 3 triangles become
//                     leaves), assigns the children to octant slots, quantises (refit.cuh: quantiseNode, the host builder's
//                     arithmetic), reserves its inner children and its triangles with two atomic counters and queues the inner
//                     children for the next level.  Levels are therefore contiguous index ranges, which is what the refit needs.
// The tree is a plain LBVH (no SAH): ~20-30 % more node visits than the host builder's tree (bvh.cpp), built in milliseconds.
// Every function is per-thread and free of warp intrinsics, so tools/host_lbvh_check.cpp runs the same source on the host.
#pragma once
#include "refit.cuh"

namespace pt {

struct LbvhWork
{
  uint32_t            m, M;       // triangles of this tree, padded to a power of two for the sort
  const float*        inRec;      // 12 floats per GLOBAL triangle (flatten order): (v0, rnode|flags<<28) (e1, prim) (e2, gid)
  const uint32_t*     subset;     // m global triangle ids (nullptr: identity)
  float4 *            primLo, *primHi;
  unsigned long long* keys;
  int *               left, *right;      // per internal node: child reference (>= 0 internal index, < 0: ~sorted leaf position)
  int *               parentI, *parentL;  // parent (internal index) of internal nodes / leaves; root: -1
  uint32_t *          first, *last;      // per internal node: range of sorted leaf positions
  float4 *            boxLo, *boxHi;     // per internal node
  uint32_t*           visits;            // per internal node: arrival counter of the bottom-up pass
  int*                cbounds;           // ordered-int min.xyz, max.xyz of the centroids
  float*              nodes;             // out: 20 floats per wide node
  float*              tris;              // out: 12 floats per triangle, leaf order
  uint32_t*           triMeta;           // out: 2 per triangle
  uint32_t            triBaseOffset;
  uint32_t*           counters;          // [0] wide nodes allocated, [1] triangles emitted, [2] entries queued for the next level
};

PT_D int      floatToOrdered(float f) { const int i = __float_as_int(f); return i >= 0 ? i : i ^ 0x7fffffff; }
PT_D float    orderedToFloat(int i) { return __int_as_float(i >= 0 ? i : i ^ 0x7fffffff); }
PT_D uint32_t globalId(const LbvhWork& W, uint32_t local) { return W.subset ? W.subset[local] : local; }

PT_D void lbvhBounds(uint32_t i, const LbvhWork& W)
{
  float lo[3], hi[3];
  triangleBox(W.inRec + (size_t)globalId(W, i) * 12, lo, hi);
  W.primLo[i] = make_float4(lo[0], lo[1], lo[2], 0.f);
  W.primHi[i] = make_float4(hi[0], hi[1], hi[2], 0.f);
  for(int a = 0; a < 3; a++)
  {
    const int c = floatToOrdered(0.5f * (lo[a] + hi[a]));
    atomicMin(&W.cbounds[a], c);
    atomicMax(&W.cbounds[3 + a], c);
  }
}

PT_D uint32_t expandBits10(uint32_t v)
{
  v = (v * 0x00010001u) & 0xFF0000FFu;
  v = (v * 0x00000101u) & 0x0F00F00Fu;
  v = (v * 0x00000011u) & 0xC30C30C3u;
  v = (v * 0x00000005u) & 0x49249249u;
  return v;
}

PT_D void lbvhMorton(uint32_t i, const LbvhWork& W)
{
  if(i >= W.m)
  {
    W.keys[i] = ~0ull;  // padding sorts to the end
    return;
  }
  uint32_t code = 0;
  for(int a = 0; a < 3; a++)
  {
    const float cmin = orderedToFloat(W.cbounds[a]), cmax = orderedToFloat(W.cbounds[3 + a]);
    const float plo[3] = {W.primLo[i].x, W.primLo[i].y, W.primLo[i].z}, phi[3] = {W.primHi[i].x, W.primHi[i].y, W.primHi[i].z};
    const float c = 0.5f * (plo[a] + phi[a]);
    const float ext = cmax - cmin;
    float       u = ext > 0.f ? (c - cmin) / ext : 0.f;
    u = fminf(fmaxf(u * 1024.f, 0.f), 1023.f);
    code |= expandBits10((uint32_t)u) << (2 - a);
  }
  W.keys[i] = ((unsigned long long)code << 32) | (unsigned long long)i;
}

// one compare-exchange of the bitonic network (thread t handles the pair (t, t ^ j) once)
PT_D void bitonicStep(uint32_t t, unsigned long long* keys, uint32_t j, uint32_t k)
{
  const uint32_t p = t ^ j;
  if(p > t)
  {
    const unsigned long long a = keys[t], b = keys[p];
    const bool               ascending = (t & k) == 0;
    if((a > b) == ascending)
    {
      keys[t] = b;
      keys[p] = a;
    }
  }
}

PT_D int lbvhDelta(const LbvhWork& W, int i, int j)
{
  if(j < 0 || j >= (int)W.m)
    return -1;
  const unsigned long long x = W.keys[i] ^ W.keys[j];
#ifdef __CUDA_ARCH__
  return __clzll((long long)x);
#else
  return x ? __builtin_clzll(x) : 64;
#endif
}

PT_D void lbvhHierarchy(uint32_t ii, const LbvhWork& W)
{
  const int i = (int)ii;
  const int d = (lbvhDelta(W, i, i + 1) - lbvhDelta(W, i, i - 1)) >= 0 ? 1 : -1;
  const int dmin = lbvhDelta(W, i, i - d);
  int       lmax = 2;
  while(lbvhDelta(W, i, i + lmax * d) > dmin)
    lmax *= 2;
  int l = 0;
  for(int t = lmax / 2; t >= 1; t /= 2)
    if(lbvhDelta(W, i, i + (l + t) * d) > dmin)
      l += t;
  const int j = i + l * d;
  const int dnode = lbvhDelta(W, i, j);
  int       s = 0, t = l;
  do
  {
    t = (t + 1) / 2;
    if(lbvhDelta(W, i, i + (s + t) * d) > dnode)
      s += t;
  } while(t > 1);
  const int gamma = i + s * d + (d < 0 ? -1 : 0);
  const int lo = i < j ? i : j, hi = i < j ? j : i;
  const int L = (lo == gamma) ? ~gamma : gamma;
  const int R = (hi == gamma + 1) ? ~(gamma + 1) : gamma + 1;
  W.left[i] = L;
  W.right[i] = R;
  W.first[i] = (uint32_t)lo;
  W.last[i] = (uint32_t)hi;
  if(L >= 0)
    W.parentI[L] = i;
  else
    W.parentL[~L] = i;
  if(R >= 0)
    W.parentI[R] = i;
  else
    W.parentL[~R] = i;
  if(i == 0)
    W.parentI[0] = -1;
}

// `fresh`: the box may have been written by another thread of the SAME launch (bottom-up fit): read it past the L1
PT_D void lbvhRefBox(const LbvhWork& W, int ref, float lo[3], float hi[3], bool fresh = false)
{
  float4 a, b;
  if(ref >= 0)
  {
#ifdef __CUDA_ARCH__
    if(fresh)
    {
      a = __ldcg(&W.boxLo[ref]);
      b = __ldcg(&W.boxHi[ref]);
    }
    else
#endif
    {
      a = W.boxLo[ref];
      b = W.boxHi[ref];
    }
  }
  else
  {
    const uint32_t prim = (uint32_t)(W.keys[~ref] & 0xffffffffull);
    a = W.primLo[prim];
    b = W.primHi[prim];
  }
  lo[0] = a.x, lo[1] = a.y, lo[2] = a.z;
  hi[0] = b.x, hi[1] = b.y, hi[2] = b.z;
}

PT_D void lbvhFit(uint32_t leaf, const LbvhWork& W)
{
  int cur = W.parentL[leaf];
  while(cur >= 0)
  {
#ifdef __CUDA_ARCH__
    __threadfence();
#endif
    if(atomicAdd(&W.visits[cur], 1u) == 0u)
      return;  // the sibling subtree is not done yet: its last thread will continue from here
#ifdef __CUDA_ARCH__
    __threadfence();
#endif
    float alo[3], ahi[3], blo[3], bhi[3];
    lbvhRefBox(W, W.left[cur], alo, ahi, true);
    lbvhRefBox(W, W.right[cur], blo, bhi, true);
    W.boxLo[cur] = make_float4(fminf(alo[0], blo[0]), fminf(alo[1], blo[1]), fminf(alo[2], blo[2]), 0.f);
    W.boxHi[cur] = make_float4(fmaxf(ahi[0], bhi[0]), fmaxf(ahi[1], bhi[1]), fmaxf(ahi[2], bhi[2]), 0.f);
    cur = W.parentI[cur];
  }
}

PT_D uint32_t lbvhRefCount(const LbvhWork& W, int ref) { return ref >= 0 ? W.last[ref] - W.first[ref] + 1u : 1u; }
PT_D uint32_t lbvhRefFirst(const LbvhWork& W, int ref) { return ref >= 0 ? W.first[ref] : (uint32_t)~ref; }

// one wide node: queueIn[q] = (binary reference, wide node index); inner children go to queueOut
PT_D void lbvhEmit(uint32_t q, const LbvhWork& W, const int2* queueIn, int2* queueOut)
{
  const int      root = queueIn[q].x;
  const uint32_t wide = (uint32_t)queueIn[q].y;
  int            ch[8];
  int            nch = 0;
  if(lbvhRefCount(W, root) <= 3u)
    ch[nch++] = root;  // (only the tree's root can be this small: it becomes a wide node with one leaf child)
  else
  {
    ch[nch++] = W.left[root];
    ch[nch++] = W.right[root];
    while(nch < 8)
    {
      int   pick = -1;
      float bestArea = -1.f;
      for(int i = 0; i < nch; i++)
      {
        if(ch[i] < 0 || lbvhRefCount(W, ch[i]) <= 3u)
          continue;
        float lo[3], hi[3];
        lbvhRefBox(W, ch[i], lo, hi);
        const float dx = hi[0] - lo[0], dy = hi[1] - lo[1], dz = hi[2] - lo[2];
        const float area = dx * dy + dy * dz + dz * dx;
        if(area > bestArea)
        {
          bestArea = area;
          pick = i;
        }
      }
      if(pick < 0)
        break;
      const int open = ch[pick];
      ch[pick] = W.left[open];
      ch[nch++] = W.right[open];
    }
  }
  // node box + child boxes
  float clo[8][3], chi[8][3], lo[3] = {3.0e38f, 3.0e38f, 3.0e38f}, hi[3] = {-3.0e38f, -3.0e38f, -3.0e38f};
  for(int i = 0; i < nch; i++)
  {
    lbvhRefBox(W, ch[i], clo[i], chi[i]);
    for(int a = 0; a < 3; a++)
    {
      lo[a] = fminf(lo[a], clo[i][a]);
      hi[a] = fmaxf(hi[a], chi[i][a]);
    }
  }
  // octant slots: slot s is visited first by rays whose direction signs are the complement of s (x -> 4, y -> 2, z -> 1);
  // greedy maximum of (child centroid - node centre) . slot diagonal
  const float cx = 0.5f * (lo[0] + hi[0]), cy = 0.5f * (lo[1] + hi[1]), cz = 0.5f * (lo[2] + hi[2]);
  int         childAt[8] = {-1, -1, -1, -1, -1, -1, -1, -1};
  bool        used[8] = {false, false, false, false, false, false, false, false};
  for(int k = 0; k < nch; k++)
  {
    float best = -3.0e38f;
    int   bi = -1, bs = -1;
    for(int i = 0; i < nch; i++)
    {
      if(used[i])
        continue;
      const float dx = 0.5f * (clo[i][0] + chi[i][0]) - cx, dy = 0.5f * (clo[i][1] + chi[i][1]) - cy, dz = 0.5f * (clo[i][2] + chi[i][2]) - cz;
      for(int s = 0; s < 8; s++)
      {
        if(childAt[s] >= 0)
          continue;
        const float c = dx * ((s & 4) ? 1.f : -1.f) + dy * ((s & 2) ? 1.f : -1.f) + dz * ((s & 1) ? 1.f : -1.f);
        if(c > best)
        {
          best = c;
          bi = i;
          bs = s;
        }
      }
    }
    used[bi] = true;
    childAt[bs] = bi;
  }
  // counts, reservations
  uint32_t innerCount = 0, triCount = 0;
  for(int s = 0; s < 8; s++)
    if(childAt[s] >= 0)
    {
      const uint32_t c = lbvhRefCount(W, ch[childAt[s]]);
      if(c <= 3u)
        triCount += c;
      else
        innerCount++;
    }
  const uint32_t childBase = innerCount ? atomicAdd(&W.counters[0], innerCount) : 0u;
  const uint32_t triLocal = triCount ? atomicAdd(&W.counters[1], triCount) : 0u;
  const uint32_t queueBase = innerCount ? atomicAdd(&W.counters[2], innerCount) : 0u;
  float          slo[8][3], shi[8][3];
  uint32_t       present = 0, imask = 0, meta[8] = {0, 0, 0, 0, 0, 0, 0, 0}, triOff = 0, innerK = 0;
  for(int s = 0; s < 8; s++)
  {
    if(childAt[s] < 0)
      continue;
    const int i = childAt[s];
    present |= 1u << s;
    for(int a = 0; a < 3; a++)
    {
      slo[s][a] = clo[i][a];
      shi[s][a] = chi[i][a];
    }
    const uint32_t c = lbvhRefCount(W, ch[i]);
    if(c > 3u)
    {
      imask |= 1u << s;
      meta[s] = (1u << 5) | (24u + (uint32_t)s);
      queueOut[queueBase + innerK] = make_int2(ch[i], (int)(childBase + innerK));
      innerK++;
    }
    else
    {
      const uint32_t bits = c == 1u ? 1u : (c == 2u ? 3u : 7u);
      meta[s] = (bits << 5) | triOff;
      const uint32_t firstLeaf = lbvhRefFirst(W, ch[i]);
      for(uint32_t k = 0; k < c; k++)
      {
        const uint32_t prim = (uint32_t)(W.keys[firstLeaf + k] & 0xffffffffull);
        const float*   src = W.inRec + (size_t)globalId(W, prim) * 12;
        const uint32_t slot = triLocal + triOff + k;
        float*         dst = W.tris + (size_t)slot * 12;
        for(int w = 0; w < 12; w++)
          dst[w] = src[w];
        W.triMeta[slot * 2] = __float_as_uint(src[3]);
        W.triMeta[slot * 2 + 1] = __float_as_uint(src[7]);
      }
      triOff += c;
    }
  }
  float* N = W.nodes + (size_t)wide * 20;
  N[3] = __uint_as_float(imask << 24);
  quantiseNode(N, lo, hi, slo, shi, present);
  N[4] = __uint_as_float(childBase | (6u << 26));  // standard axis map: slot bit 0 -> z, 1 -> y, 2 -> x
  N[5] = __uint_as_float(W.triBaseOffset + triLocal);
  N[6] = __uint_as_float(meta[0] | (meta[1] << 8) | (meta[2] << 16) | (meta[3] << 24));
  N[7] = __uint_as_float(meta[4] | (meta[5] << 8) | (meta[6] << 16) | (meta[7] << 24));
}

}  // namespace pt
