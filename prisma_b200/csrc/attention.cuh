// prisma_b200 -- ViT attention launch descriptor (see attention.cu).
#pragma once
#include "common.cuh"

namespace prisma {

struct AttnArgs {
  int tokens, heads, D, batch;
  __half* out;
  int out_ld;
};
struct AttnLaunch {
  CUtensorMap tm;
  AttnArgs args;
  dim3 grid;
  double flops = 0;
};
// qkv fp16 [batch*tokens][3*D] (q rows pre-scaled by 1/sqrt(64)) -> out fp16 [batch*tokens][D]
int attention_prepare(AttnLaunch* out, const __half* qkv, __half* o, int batch, int tokens, int heads, int D);
int attention_run(const AttnLaunch& a, cudaStream_t s);

}  // namespace prisma
