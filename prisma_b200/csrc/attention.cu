// prisma_b200 -- ViT self-attention on wgmma (sm_90a): softmax(q k^T) v, non-causal, head_dim 64
// (dinov2/layers/attention.py:49-62; the 1/sqrt(64) scale is folded into the q rows of the qkv weights, exactly).
//
// One CTA per (128-query tile, head, image):
//   warp 8        : TMA producer  (Q once; K/V 128x64 fp16 tiles in a 2-stage ring, 128B swizzle, straight out of the
//                                  [tokens][3*D] qkv matrix -- no head split / transposes ever materialise)
//   warpgroups 0-1: 64 query rows each.  S = Q K^T (wgmma m64n128k16, both operands from shared memory) lands in registers;
//                   the online softmax runs on that fragment (a row is spread over the 4 lanes of a quad); P is repacked to
//                   fp16 in registers -- the accumulator layout of two 8-column blocks IS the A-operand layout of one
//                   K = 16 step -- and O += P V (wgmma m64n64k16, A from registers, V from shared memory as an MN-major
//                   operand) accumulates in registers.  P never goes through shared memory.  The two warpgroups run
//                   independently, so one's softmax overlaps the other's MMAs.
#include "attention.cuh"
#include "wgmma.cuh"

namespace prisma {

constexpr int ATT_BQ = 128, ATT_BKV = 128, ATT_HD = 64;
constexpr int ATT_THREADS = 288;  // 2 consumer warpgroups + 1 producer warp
constexpr int ATT_TILE_BYTES = 128 * 64 * 2;  // 16 KB
// Q + 2 x (K, V) + barriers; the dynamic smem base is declared 1024-aligned (128B-swizzle atoms are 1 KB) and checked at entry
constexpr int ATT_SMEM = ATT_TILE_BYTES * (1 + 2 + 2) + 128 /*barriers*/;

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

__global__ void __launch_bounds__(ATT_THREADS, 1)
attention_kernel(const __grid_constant__ CUtensorMap tmQKV, const __grid_constant__ AttnArgs args) {
  extern __shared__ __align__(1024) uint8_t smem[];
  if ((smem_u32(smem) & 1023u) != 0) __trap();  // 128B-swizzle atoms are 1 KB
  uint8_t* sQ = smem;
  uint8_t* sK = smem + ATT_TILE_BYTES;      // 2 stages
  uint8_t* sV = smem + 3 * ATT_TILE_BYTES;  // 2 stages
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + 5 * ATT_TILE_BYTES);
  uint64_t* q_full = bars + 0;
  uint64_t* kv_full = bars + 1;   // [2]
  uint64_t* kv_empty = bars + 3;  // [2]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int T = args.tokens, D = args.D;
  const int q0 = blockIdx.x * ATT_BQ;
  const int head = blockIdx.y;
  const int row_base = blockIdx.z * T;  // first row of this image in the qkv matrix
  const int n_kv = (T + ATT_BKV - 1) / ATT_BKV;

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmQKV);
    mbar_init(q_full, 1);
    for (int s = 0; s < 2; ++s) { mbar_init(&kv_full[s], 1); mbar_init(&kv_empty[s], 2); }  // one arrival per warpgroup
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == 8) {
    if (lane == 0) {
      mbar_arrive_expect_tx(q_full, ATT_TILE_BYTES);
      tma_load_2d(sQ, &tmQKV, q_full, head * ATT_HD, row_base + q0);
      for (int j = 0; j < n_kv; ++j) {
        const int st = j & 1;
        mbar_wait(&kv_empty[st], ((j >> 1) & 1) ^ 1);
        mbar_arrive_expect_tx(&kv_full[st], 2 * ATT_TILE_BYTES);
        tma_load_2d(sK + st * ATT_TILE_BYTES, &tmQKV, &kv_full[st], D + head * ATT_HD, row_base + j * ATT_BKV);
        tma_load_2d(sV + st * ATT_TILE_BYTES, &tmQKV, &kv_full[st], 2 * D + head * ATT_HD, row_base + j * ATT_BKV);
      }
    }
    return;
  }

  const int wg = warp >> 2;
  const int tq = lane & 3;
  const float LOG2E = 1.4426950408889634f;
  const uint64_t qdesc = make_wgmma_desc(smem_u32(sQ + wg * 64 * 128));
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_sum[2] = {0.f, 0.f};  // rows r and r + 8 of this thread
  mbar_wait(q_full, 0);

  for (int j = 0; j < n_kv; ++j) {
    const int st = j & 1;
    mbar_wait(&kv_full[st], (j >> 1) & 1);
    float s[64];
    const uint64_t kdesc = make_wgmma_desc(smem_u32(sK + st * ATT_TILE_BYTES));
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) Wgmma<128>::f16(s, qdesc + 2 * k, kdesc + 2 * k, k != 0);
    wgmma_commit();
    wgmma_wait<0>();

    // keys beyond the last token of the image (last KV tile) do not take part
    const int valid = min(ATT_BKV, T - j * ATT_BKV);
    if (valid < ATT_BKV) {
#pragma unroll
      for (int jj = 0; jj < 16; ++jj) {
        const int c = jj * 8 + tq * 2;
        if (c >= valid) { s[jj * 4] = -INFINITY; s[jj * 4 + 2] = -INFINITY; }
        if (c + 1 >= valid) { s[jj * 4 + 1] = -INFINITY; s[jj * 4 + 3] = -INFINITY; }
      }
    }
    // ---- row max over the quad, rescale of O and l
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int jj = 0; jj < 16; ++jj) {
      mx[0] = fmaxf(mx[0], fmaxf(s[jj * 4], s[jj * 4 + 1]));
      mx[1] = fmaxf(mx[1], fmaxf(s[jj * 4 + 2], s[jj * 4 + 3]));
    }
    float msc[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
      mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
      const float m_new = fmaxf(fmaxf(m_run[h], mx[h]), -60000.f);  // a row of -inf scores must not produce inf - inf
      const float alpha = ex2_approx((m_run[h] - m_new) * LOG2E);   // 0 on the first tile
      l_sum[h] *= alpha;
#pragma unroll
      for (int d = 0; d < 8; ++d) { o[d * 4 + 2 * h] *= alpha; o[d * 4 + 2 * h + 1] *= alpha; }
      m_run[h] = m_new;
      msc[h] = m_new * LOG2E;
    }
    // ---- p = exp(s - m), row sums, fp16 A fragments of the PV product
    uint32_t pa[8][4];
#pragma unroll
    for (int jj = 0; jj < 16; ++jj) {
      const float p0 = ex2_approx(fmaf(s[jj * 4], LOG2E, -msc[0])), p1 = ex2_approx(fmaf(s[jj * 4 + 1], LOG2E, -msc[0]));
      const float p2 = ex2_approx(fmaf(s[jj * 4 + 2], LOG2E, -msc[1])), p3 = ex2_approx(fmaf(s[jj * 4 + 3], LOG2E, -msc[1]));
      l_sum[0] += p0 + p1;
      l_sum[1] += p2 + p3;
      pa[jj >> 1][(jj & 1) * 2] = pack_half2(p0, p1);
      pa[jj >> 1][(jj & 1) * 2 + 1] = pack_half2(p2, p3);
    }
    // ---- O += P V: 8 K-steps of 16 keys; V rows (keys) are 128 B = 64 head dims: MN-major B, 2 KB per step
    const uint32_t vbase = smem_u32(sV + st * ATT_TILE_BYTES);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) Wgmma<64>::f16_rs_bmn(o, pa[kk], make_wgmma_desc(vbase + kk * 2048), 1);
    wgmma_commit();
    wgmma_wait<0>();
    if ((threadIdx.x & 127) == 0) mbar_arrive(&kv_empty[st]);
  }

  // ---- normalise and store: rows r (o[4d], o[4d+1]) and r + 8 (o[4d+2], o[4d+3]), columns 8d + 2 tq
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    l_sum[h] += __shfl_xor_sync(0xffffffffu, l_sum[h], 1);
    l_sum[h] += __shfl_xor_sync(0xffffffffu, l_sum[h], 2);
    const float inv = 1.0f / l_sum[h];
    const int q = q0 + wg * 64 + (warp & 3) * 16 + (lane >> 2) + h * 8;
    if (q < T) {
      __half* dst = args.out + (size_t)(row_base + q) * args.out_ld + head * ATT_HD + tq * 2;
#pragma unroll
      for (int d = 0; d < 8; ++d)
        *reinterpret_cast<uint32_t*>(dst + d * 8) = pack_half2(o[d * 4 + 2 * h] * inv, o[d * 4 + 2 * h + 1] * inv);
    }
  }
}

int attention_prepare(AttnLaunch* out, const __half* qkv, __half* o, int batch, int tokens, int heads, int D) {
  PRISMA_CHECK(D == heads * ATT_HD, "attention: head_dim must be 64");
  out->args.tokens = tokens;
  out->args.heads = heads;
  out->args.D = D;
  out->args.batch = batch;
  out->args.out = o;
  out->args.out_ld = D;
  PRISMA_TRY(make_tmap_2d_f16(&out->tm, qkv, (uint64_t)3 * D, (uint64_t)batch * tokens, (uint64_t)3 * D, 64, 128));
  out->grid = dim3(ceil_div(tokens, ATT_BQ), heads, batch);
  out->flops = 4.0 * batch * heads * (double)tokens * tokens * ATT_HD;
  return 0;
}

int attention_run(const AttnLaunch& a, cudaStream_t s) {
  static bool attr_set = false;
  if (!attr_set) {
    PRISMA_CUDA_OK(cudaFuncSetAttribute(attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, ATT_SMEM));
    attr_set = true;
  }
  attention_kernel<<<a.grid, ATT_THREADS, ATT_SMEM, s>>>(a.tm, a.args);
  PRISMA_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace prisma
