// host_dlss_check.cpp — the device DLSS arithmetic (dlss_guides.cuh: dlssEnvBRDFApprox2, dlssMotionVector, the binary16 and
// UNORM8 conversions) compiled for the host and run on records written by tests/test_dlss_guides.py.
//   host_dlss_check brdf   in.bin out.bin   in: f32 [n][5] (specular colour xyz, alpha, NoV)          out: f32 [n][3]
//   host_dlss_check motion in.bin out.bin   in: f32 prevMVP[16], currMVP[16], [n][10] (curr, prev, res) out: f32 [n][2]
//   host_dlss_check pack   in.bin out.bin   in: f32 [n]                                               out: u16 half[n], u32 unorm8[n]
#include "host_shim.h"

#include <cstdio>
#include <cstring>
#include <vector>

#include "../dlss_guides.cuh"

using namespace pt;

int main(int argc, char** argv)
{
  if(argc < 4)
    return 2;
  FILE* f = std::fopen(argv[2], "rb");
  if(!f)
    return 2;
  std::vector<float> in;
  float              v;
  while(std::fread(&v, 4, 1, f) == 1)
    in.push_back(v);
  std::fclose(f);
  FILE* o = std::fopen(argv[3], "wb");
  if(!o)
    return 2;
  if(!std::strcmp(argv[1], "brdf"))
  {
    for(size_t i = 0; i + 5 <= in.size(); i += 5)
    {
      const float3 r = dlssEnvBRDFApprox2(f3(in[i], in[i + 1], in[i + 2]), in[i + 3], in[i + 4]);
      std::fwrite(&r, 4, 3, o);
    }
  }
  else if(!std::strcmp(argv[1], "motion"))
  {
    if(in.size() < 32)
      return 2;
    for(size_t i = 32; i + 10 <= in.size(); i += 10)
    {
      const float* p = &in[i];
      const float2 mv = dlssMotionVector(f4(p[0], p[1], p[2], p[3]), f4(p[4], p[5], p[6], p[7]), &in[0], &in[16], f2(p[8], p[9]));
      std::fwrite(&mv, 4, 2, o);
    }
  }
  else if(!std::strcmp(argv[1], "pack"))
  {
    for(float x : in)
    {
      const uint16_t h = dlssHalfBits(x);
      std::fwrite(&h, 2, 1, o);
    }
    for(float x : in)
    {
      const uint32_t u = dlssUnorm8(x);
      std::fwrite(&u, 4, 1, o);
    }
  }
  else
    return 2;
  std::fclose(o);
  return 0;
}
