// host_phase_check.cpp — the device Henyey-Greenstein phase function (../bsdf.cuh: sampleHenyeyGreenstein,
// henyeyGreensteinPdf) compiled for the host through host_shim.h and run on records written by tests/test_phase_sampling.py.
//   host_phase_check sample in.bin out.bin   in: f32 [n][6] (xi.x, xi.y, g, wi xyz)   out: f32 [n][3]
//   host_phase_check pdf    in.bin out.bin   in: f32 [n][2] (cos theta, g)           out: f32 [n]
#include "host_shim.h"

#include <cstdio>
#include <cstring>
#include <vector>

#include "../bsdf.cuh"

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
  if(!std::strcmp(argv[1], "sample"))
  {
    for(size_t i = 0; i + 6 <= in.size(); i += 6)
    {
      const float3 d = sampleHenyeyGreenstein(f2(in[i], in[i + 1]), in[i + 2], f3(in[i + 3], in[i + 4], in[i + 5]));
      std::fwrite(&d, 4, 3, o);
    }
  }
  else if(!std::strcmp(argv[1], "pdf"))
  {
    for(size_t i = 0; i + 2 <= in.size(); i += 2)
    {
      const float p = henyeyGreensteinPdf(in[i], in[i + 1]);
      std::fwrite(&p, 4, 1, o);
    }
  }
  else
    return 2;
  std::fclose(o);
  return 0;
}
