// bvh_stats.cpp — offline (CPU) quality check of the wide-BVH builder: traverses the compressed tree exactly like
// the CUDA kernel (same decode, same octant order, closest-hit culling by best t) and reports nodes / triangles
// visited per ray.  Input: a binary dump written by scripts/dump_bvh_input.py:
//   u32 nTris, u32 nRays, nTris x 9 floats (v0,e1,e2), nRays x 8 floats (o,tmin,d,tmax)
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../bvh.h"
using namespace pt;

static inline uint32_t fu(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }
static inline float    uf(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }

int main(int argc, char** argv)
{
  if(argc < 2) { fprintf(stderr, "usage: bvh_stats dump.bin\n"); return 1; }
  FILE* f = fopen(argv[1], "rb");
  uint32_t nT, nR;
  if(fread(&nT, 4, 1, f) != 1 || fread(&nR, 4, 1, f) != 1) return 1;
  std::vector<float> tv((size_t)nT * 9), rv((size_t)nR * 8);
  if(fread(tv.data(), 4, tv.size(), f) != tv.size() || fread(rv.data(), 4, rv.size(), f) != rv.size()) return 1;
  fclose(f);
  std::vector<FlatTri> tris(nT);
  std::vector<uint32_t> gids(nT);
  for(uint32_t i = 0; i < nT; i++)
  {
    memcpy(tris[i].v0, &tv[i * 9], 12); memcpy(tris[i].e1, &tv[i * 9 + 3], 12); memcpy(tris[i].e2, &tv[i * 9 + 6], 12);
    tris[i].rnode = 0; tris[i].prim = i; tris[i].flags = TRI_OPAQUE | TRI_NOCULL; gids[i] = i;
  }
  WideBvh B;
  buildWideBvh(tris, gids, 0, B);
  printf("tris %u nodes %u (%.1f MB nodes, %.1f MB tris) depth %u\n", B.numTris, B.numNodes, B.nodes.size() * 4 / 1e6, B.tris.size() * 4 / 1e6, B.maxDepth);
  double nodes = 0, tt = 0, hits = 0;
  for(uint32_t r = 0; r < nR; r++)
  {
    const float* R = &rv[r * 8];
    float org[3] = {R[0], R[1], R[2]}, dir[3] = {R[4], R[5], R[6]}, tmin = R[3], best = R[7];
    float id[3];
    for(int a = 0; a < 3; a++) { float d = fabsf(dir[a]) > 1e-20f ? dir[a] : copysignf(1e-20f, dir[a]); id[a] = 1.0f / d; }
    const uint32_t dsign = (dir[0] < 0 ? 0 : 1) | (dir[1] < 0 ? 0 : 2) | (dir[2] < 0 ? 0 : 4);
    struct G { uint32_t x, y; };
    G stack[64]; int sp = 0; G cur{0, 0x80000000u};
    bool hit = false;
    for(;;)
    {
      G tg{0, 0};
      if(cur.y & 0xff000000u)
      {
        uint32_t him = cur.y; int cb = 31 - __builtin_clz(him);
        cur.y &= ~(1u << cb);
        if(cur.y & 0xff000000u) stack[sp++] = cur;
        uint32_t slot = (uint32_t)(cb - 24) ^ ((him >> 8) & 7u);
        uint32_t rel = __builtin_popcount(him & ~(0xffffffffu << slot));
        const float* N = &B.nodes[(size_t)(cur.x + rel) * 20];
        nodes++;
        uint32_t eim = fu(N[3]);
        float ad[3], ao[3];
        for(int a = 0; a < 3; a++) { ad[a] = uf(((eim >> (8 * a)) & 0xff) << 23) * id[a]; ao[a] = (N[a] - org[a]) * id[a]; }
        const uint32_t amap = fu(N[4]) >> 26;
        const uint32_t octInv = ((dsign >> (amap & 3)) & 1) | (((dsign >> ((amap >> 2) & 3)) & 1) << 1) | (((dsign >> (amap >> 4)) & 1) << 2);
        cur.x = fu(N[4]) & 0x03ffffffu; tg.x = fu(N[5]);
        uint32_t hm = 0;
        for(int c = 0; c < 8; c++)
        {
          uint32_t meta = (fu(N[6 + c / 4]) >> (8 * (c % 4))) & 0xff;
          bool inner = (meta & (meta << 1)) & 0x10;
          uint32_t bitIndex = (meta ^ (inner ? octInv : 0)) & 0x1f, childBits = (meta >> 5) & 7;
          float tn = tmin, tf = best;
          for(int a = 0; a < 3; a++)
          {
            uint32_t lo = (fu(N[8 + a * 4 + c / 4]) >> (8 * (c % 4))) & 0xff, hi = (fu(N[8 + a * 4 + 2 + c / 4]) >> (8 * (c % 4))) & 0xff;
            float t0 = (dir[a] < 0 ? hi : lo) * ad[a] + ao[a], t1 = (dir[a] < 0 ? lo : hi) * ad[a] + ao[a];
            tn = fmaxf(tn, t0); tf = fminf(tf, t1);
          }
          if(tn <= tf * 1.000001f) hm |= childBits << bitIndex;
        }
        cur.y = (hm & 0xff000000u) | (octInv << 8) | (eim >> 24); tg.y = hm & 0x00ffffffu;
      }
      else { tg = cur; cur = G{0, 0}; }
      while(tg.y)
      {
        int tb = 31 - __builtin_clz(tg.y); tg.y &= ~(1u << tb);
        const float* T = &B.tris[(size_t)(tg.x + tb) * 12];
        tt++;
        float e1[3] = {T[4], T[5], T[6]}, e2[3] = {T[8], T[9], T[10]};
        float p[3] = {dir[1] * e2[2] - dir[2] * e2[1], dir[2] * e2[0] - dir[0] * e2[2], dir[0] * e2[1] - dir[1] * e2[0]};
        float det = e1[0] * p[0] + e1[1] * p[1] + e1[2] * p[2];
        if(det == 0) continue;
        float inv = 1 / det, tv3[3] = {org[0] - T[0], org[1] - T[1], org[2] - T[2]};
        float u = (tv3[0] * p[0] + tv3[1] * p[1] + tv3[2] * p[2]) * inv;
        if(u < 0 || u > 1) continue;
        float q[3] = {tv3[1] * e1[2] - tv3[2] * e1[1], tv3[2] * e1[0] - tv3[0] * e1[2], tv3[0] * e1[1] - tv3[1] * e1[0]};
        float v = (dir[0] * q[0] + dir[1] * q[1] + dir[2] * q[2]) * inv;
        if(v < 0 || u + v > 1) continue;
        float t = (e2[0] * q[0] + e2[1] * q[1] + e2[2] * q[2]) * inv;
        if(t > tmin && t < best) { best = t; hit = true; }
      }
      if((cur.y & 0xff000000u) == 0) { if(sp == 0) break; cur = stack[--sp]; }
    }
    hits += hit;
  }
  printf("rays %u: %.2f nodes/ray, %.2f tris/ray, hit rate %.3f\n", nR, nodes / nR, tt / nR, hits / nR);
  return 0;
}
