// prisma_b200 -- the wgmma "shifted-row GEMM" core (sm_90a).
//
//   D[m, n] = sum_{t < taps} sum_{c < Cin} A[m + tap_off[t], c] * W[n, t * kchunks*64 + c]        (fp16 x fp16 -> fp32)
//
// taps == 1, tap_off = {0}  : a plain GEMM (ViT linears, 1x1 convs, transposed convs with k == s, RAFT correlation)
// taps == kh*kw             : an implicit-GEMM convolution over a zero-bordered NHWC activation whose pixels are
//                             flattened to rows; tap (ky,kx) is the same 2-D TMA box shifted by (ky-ph)*Wp + (kx-pw)
//                             rows.  Border rows are computed and discarded (waste 2/(W+2)); no im2col buffer, no 4-D
//                             tensor map; TMA zero-fills out-of-range rows (either sign).
//
// Kernel anatomy (persistent, warp-specialised, one CTA per SM, 384 threads):
//   warpgroups 0-1 : consumers  (each: wgmma.mma_async M=64 x N=BN x K=16 over its 64 rows of the 128-row tile, fp32
//                                accumulators in registers; then the epilogue of those rows)
//   warpgroup  2   : producer   (one thread: TMA loads of A 128x64 and W BNx64 fp16 tiles, 128B swizzle, STAGES-deep
//                                mbarrier ring; its registers are handed to the consumers with setmaxnreg)
// Epilogue: a warp holds 16 accumulator rows; the two warps of a pair (32 consecutive rows) exchange their fragments through
// their swizzled 32 x 32 fp32 staging buffers, so that each then owns one 32-row x 32-column chunk and applies bias / GELU /
// ReLU / LayerScale / residuals with coalesced fp32 and/or fp16 stores in the row mapping of the consumer's layout (every
// global access of a chunk is issued as a batch of 8 independent requests per lane), or stores it with TMA.
#pragma once
#include "common.cuh"
#include "wgmma.cuh"

namespace prisma {

constexpr int GEMM_BM = 128;
constexpr int GEMM_BK = 64;
constexpr int GEMM_THREADS = 384;                           // 2 consumer warpgroups + 1 producer warpgroup
constexpr int GEMM_SMEM_MAX = 232448;                       // 227 KB of dynamic shared memory per CTA
constexpr int GEMM_MAX_TAPS = 49;

enum RowMap : int {
  ROW_LINEAR = 0,   // dst row = m                                   (valid: m < M)
  ROW_PADDED = 1,   // m indexes a zero-bordered [Hp][Wp] image; only interior pixels are stored (borders stay zero)
  ROW_TOK2PAD = 2,  // m = y*W + x (dense tokens)  -> dst row (y+1)*out_wp + x+1
  ROW_PAD2TOK = 5,  // m indexes a zero-bordered image; interior pixel (y,x) -> dense dst row img*H*W + y*W + x
  ROW_TOKSKIP = 4,  // m = b*P + p (patch tokens of image b) -> dst row b*(P+1) + 1 + p  (skips the cls rows; in_w = P)
  ROW_SHUFFLE = 3,  // ConvTranspose k == s: m = y*W + x, n = (dy*s+dx)*cout + co -> dst row (y*s+dy+1)*out_wp + x*s+dx+1
};

struct GemmEpilogue {
  float alpha = 1.0f;            // accumulator scale (e.g. 1/sqrt(C) of the RAFT correlation), applied first
  const float* bias = nullptr;   // [N]
  const float* gamma = nullptr;  // [N]  LayerScale
  int act = 0;                   // 0 none, 1 exact-erf GELU, 2 ReLU, 3 sigmoid, 4 tanh (fast, ~4e-7), 5 softplus, 6 sigmoid (expf + IEEE div)
  const float* pre_f32 = nullptr;  // + a per-element fp32 term BEFORE the activation, indexed by dst row (e.g. the part of a
  int pre_f32_ld = 0;              //   conv over concatenated inputs that does not change between iterations)
  const float* res_f32 = nullptr;  // + residual (fp32), indexed by dst row
  int res_f32_ld = 0;
  const __half* res_a = nullptr;  // + residual (fp16), indexed by dst row
  int res_a_ld = 0;
  const __half* res_b = nullptr;
  int res_b_ld = 0;
  float* out_f32 = nullptr;
  int out_f32_ld = 0;
  __half* out_f16 = nullptr;
  int out_f16_ld = 0;
  __half* out_f16_relu = nullptr;  // relu(result) copy, for consumers that take relu(x) as operand and x as skip
  int out_f16_relu_ld = 0;
  int row_map = ROW_LINEAR;
  int img_rows = 0;  // ROW_PADDED: rows per image (Hp*Wp); 0 = single image
  int in_w = 0;      // ROW_PADDED: Wp ; ROW_TOK2PAD / ROW_SHUFFLE: W
  int in_h = 0;      // ROW_PADDED: Hp ; ROW_TOK2PAD / ROW_SHUFFLE: H (rows per image = H*W)
  int out_wp = 0;    // destination padded width
  int out_img_rows = 0;  // destination rows per image
  int sub = 1;       // ROW_PADDED: keep every sub-th pixel (stride-2 conv evaluated at stride 1)
  int pad = 1;       // ROW_PADDED / ROW_PAD2TOK: border width of the input geometry; out_pad: of the destination
  int out_pad = 1;
  // Border placement.  lead < 0 (default): symmetric border, `pad` pixels on every side (in_h = H + 2 pad).
  // lead == 0: "shared border" layout -- `pad` zero columns only at the END of every row and `pad` zero rows only at the END
  // of every image (in_h = H + pad, in_w = W + pad).  A negative tap shift then lands in the previous row's / previous
  // image's trailing zeros (or before row 0, where TMA zero-fills), so the halo is still all zeros but the GEMM walks
  // (H + pad)(W + pad) rows instead of (H + 2 pad)(W + 2 pad).  out_lead: the same for the destination map.
  int lead = -1;
  int out_lead = -1;
  int shuf_s = 1;
  int shuf_cout = 0;
  // fused DPT output head (dpt.py:96-100): depth = relu(head_b + sum_j head_w[j] * relu(acc[j] + bias[j])), N == 32,
  // written dense fp32 [H][W] (ROW_PADDED input geometry)
  const float* head_w = nullptr;
  float head_b = 0.f;
  float* head_out = nullptr;
  // Column statistics of the stored values, for a normalisation that follows the conv (RAFT's InstanceNorm2d): every
  // 32-row slab of the output space (slab = m / 32; image row counts are multiples of 32, so a slab lies in one image)
  // writes sum and sum of squares over its VALID rows: stat_part[(slab * 2 + {0,1}) * N + n], fp32, deterministic
  // (fixed shuffle tree; a second kernel adds the slabs in double precision in a fixed order).
  float* stat_part = nullptr;
  // Row count known only on the device (SOLOv2: the number of candidates of this frame): when set, only the first
  // round_up(*m_dev, 128) rows of the output space are computed (the launch is sized for the capacity M).
  const int* m_dev = nullptr;
  // dense output (row_map LINEAR; out_f32: scale, bias, LayerScale; out_f16: scale, bias, GELU / ReLU) stored by TMA:
  // accumulator registers -> swizzled smem box -> cp.async.bulk.tensor
  bool tma_store = false;
  // set by gemm_prepare when tma_store is asked for an in-place fp32 residual update (res_f32 == out_f32: the ViT proj / fc2
  // linears, x += gamma (acc + bias)): the staged box leaves through cp.reduce.async.bulk.tensor ... .add.f32 -- the add is
  // done by the L2 (one round-to-nearest fp32 add per element, as the register path does); the epilogue reads nothing
  bool tma_reduce = false;
  // ConvGRU gate arithmetic in the epilogue of the gate convs (raft/update.py:54-58), all fp32, indexed by dst row:
  //  gru == 1 (the z | r conv, N = 256, act sigmoid): columns [0,128) = z -> out_f32 as usual; columns [128,256) = r are not
  //            stored: r * h (gru_h: fp32 [rows][128]) goes to gru_rh (fp16, pitch gru_rh_ld) -- the q conv's operand;
  //  gru == 2 (the q conv, N = 128, act tanh): h' = (1 - z) h + z q with z = gru_z (fp32, pitch 256) and h = gru_h; h' then
  //            takes the normal output path (out_f32 = the fp32 master of h, in place; out_f16 = the conv operand copy).
  int gru = 0;
  const float* gru_h = nullptr;
  const float* gru_z = nullptr;
  __half* gru_rh = nullptr;
  int gru_rh_ld = 0;
};

struct GemmArgs {
  int M;  // rows of the output space
  int N;  // output columns
  int taps;
  int kchunks;  // 64-wide K blocks per tap
  int tap_off[GEMM_MAX_TAPS];
  int tap_acol[GEMM_MAX_TAPS];  // first A column (elements) of each tap's K slab: 0 for plain convs; the 3xTF32 path walks
                                // [hi | lo] activation halves: (hi, W_hi), (lo, W_hi), (hi, W_lo)
  int acc_group;  // XACC kernels: K blocks accumulated inside one wgmma chain before the partial sum is added to the running
                  // fp32 sums with round-to-nearest FADDs (see gemm_prepare_tf32x3)
  int raster_n;  // 1: consecutive tiles walk N first (the CTAs of a wave share few A row panels and all of W: A is read
                 // from HBM once when M >> N); 0: M first
  GemmEpilogue ep;
};

template <int BN, bool TMAST = false>  // TMAST: TMA-store epilogue (double-buffered staging boxes)
struct GemmCfg {
  static constexpr int A_BYTES = GEMM_BM * GEMM_BK * 2;  // 128 rows x 128 B (64 fp16, or 32 fp32 on the tf32 path)
  static constexpr int B_BYTES = BN * GEMM_BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int STG_WARP = TMAST ? 8192 : 4096;     // per consumer warp: one (two) 32 x 128 B boxes
  static constexpr int STG_BYTES = 8 * STG_WARP;
  static constexpr int FIT = (GEMM_SMEM_MAX - STG_BYTES - 1280) / STAGE_BYTES;  // operand stages that fit beside the staging
  static constexpr int STAGES = FIT > 8 ? 8 : FIT;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + STG_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
  static_assert(STAGES >= 3, "too few operand stages");
};

#ifdef __CUDACC__
__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752f)); }
// sigmoid / tanh of the fused epilogues: ex2.approx + rcp.approx (relative error ~4e-7, absolute error of tanh ~2e-7) instead
// of expf + IEEE division / tanhf: far fewer instructions per element, and their accuracy is irrelevant next to the fp16
// operand rounding (~5e-4).
__device__ __forceinline__ float sigmoid_f(float x) { return __fdividef(1.0f, 1.0f + __expf(-x)); }
__device__ __forceinline__ float tanh_f(float x) { return 1.0f - __fdividef(2.0f, __expf(2.0f * x) + 1.0f); }
__device__ __forceinline__ float softplus_f(float x) { return x > 20.f ? x : log1pf(expf(x)); }  // nn.Softplus(beta 1, threshold 20)

__device__ __forceinline__ float4 lds128(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
  return v;
}
__device__ __forceinline__ void sts128(uint32_t addr, float a, float b, float c, float d) {
  asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}
__device__ __forceinline__ void add_h4(float4& v, const uint2& r) {
  const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&r.x));
  const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&r.y));
  v.x += a.x; v.y += a.y; v.z += b.x; v.w += b.y;
}

// Coalesced phase of the epilogue for one 32-column chunk: this lane owns 4 consecutive columns (col..col+3) of the
// 8 rows dr[0..7] (8 lanes cover a row's 32 columns, so a warp instruction touches 4 rows x 128 B fp32 / 64 B fp16).
// All loads of a kind are issued before any is consumed (8 independent requests in flight per lane).
template <bool GRU>  // GRU: compile the ConvGRU gate paths (fp16-operand instantiations only; keeps the 3xTF32 kernels lean)
__device__ __forceinline__ void epilogue_rows8(const GemmEpilogue& ep, float4 (&v)[8], const int (&dr)[8], uint32_t okm,
                                               const float4& bias, const float4& gamma, int col) {
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    v[i].x = fmaf(v[i].x, ep.alpha, bias.x); v[i].y = fmaf(v[i].y, ep.alpha, bias.y);
    v[i].z = fmaf(v[i].z, ep.alpha, bias.z); v[i].w = fmaf(v[i].w, ep.alpha, bias.w);
  }
  if (ep.pre_f32) {
    float4 t[8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
      t[i] = (okm >> i) & 1 ? *reinterpret_cast<const float4*>(ep.pre_f32 + (size_t)dr[i] * ep.pre_f32_ld + col)
                            : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int i = 0; i < 8; ++i) { v[i].x += t[i].x; v[i].y += t[i].y; v[i].z += t[i].z; v[i].w += t[i].w; }
  }
  if (ep.act == 1) {
#pragma unroll
    for (int i = 0; i < 8; ++i) { v[i].x = gelu_erf(v[i].x); v[i].y = gelu_erf(v[i].y); v[i].z = gelu_erf(v[i].z); v[i].w = gelu_erf(v[i].w); }
  } else if (ep.act == 2) {
#pragma unroll
    for (int i = 0; i < 8; ++i) { v[i].x = fmaxf(v[i].x, 0.f); v[i].y = fmaxf(v[i].y, 0.f); v[i].z = fmaxf(v[i].z, 0.f); v[i].w = fmaxf(v[i].w, 0.f); }
  } else if (ep.act == 3) {
#pragma unroll
    for (int i = 0; i < 8; ++i) { v[i].x = sigmoid_f(v[i].x); v[i].y = sigmoid_f(v[i].y); v[i].z = sigmoid_f(v[i].z); v[i].w = sigmoid_f(v[i].w); }
  } else if (ep.act == 4) {
#pragma unroll
    for (int i = 0; i < 8; ++i) { v[i].x = tanh_f(v[i].x); v[i].y = tanh_f(v[i].y); v[i].z = tanh_f(v[i].z); v[i].w = tanh_f(v[i].w); }
  } else if (ep.act == 6) {  // sigmoid with expf and an IEEE division: the mask predictions of the fp32-class SOLOv2 head
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      v[i].x = 1.0f / (1.0f + expf(-v[i].x)); v[i].y = 1.0f / (1.0f + expf(-v[i].y));
      v[i].z = 1.0f / (1.0f + expf(-v[i].z)); v[i].w = 1.0f / (1.0f + expf(-v[i].w));
    }
  } else if (ep.act == 5) {
#pragma unroll
    for (int i = 0; i < 8; ++i) { v[i].x = softplus_f(v[i].x); v[i].y = softplus_f(v[i].y); v[i].z = softplus_f(v[i].z); v[i].w = softplus_f(v[i].w); }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) { v[i].x *= gamma.x; v[i].y *= gamma.y; v[i].z *= gamma.z; v[i].w *= gamma.w; }
  if (GRU && ep.gru == 1) {
    if (col >= 128) {  // warp-uniform: a 32-column chunk lies in one half
      float4 h[8];
#pragma unroll
      for (int i = 0; i < 8; ++i)
        h[i] = (okm >> i) & 1 ? *reinterpret_cast<const float4*>(ep.gru_h + (size_t)dr[i] * 128 + (col - 128))
                              : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int i = 0; i < 8; ++i)
        if ((okm >> i) & 1)
          *reinterpret_cast<uint2*>(ep.gru_rh + (size_t)dr[i] * ep.gru_rh_ld + (col - 128)) =
              make_uint2(pack_half2(v[i].x * h[i].x, v[i].y * h[i].y), pack_half2(v[i].z * h[i].z, v[i].w * h[i].w));
      return;
    }
  } else if (GRU && ep.gru == 2) {
    float4 z[8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
      z[i] = (okm >> i) & 1 ? *reinterpret_cast<const float4*>(ep.gru_z + (size_t)dr[i] * 256 + col) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int i = 0; i < 8; ++i) { v[i].x *= z[i].x; v[i].y *= z[i].y; v[i].z *= z[i].z; v[i].w *= z[i].w; }   // z q
#pragma unroll
    for (int i = 0; i < 8; ++i) { z[i].x = 1.f - z[i].x; z[i].y = 1.f - z[i].y; z[i].z = 1.f - z[i].z; z[i].w = 1.f - z[i].w; }
    float4 h[8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
      h[i] = (okm >> i) & 1 ? *reinterpret_cast<const float4*>(ep.gru_h + (size_t)dr[i] * 128 + col) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int i = 0; i < 8; ++i) {  // (1 - z) * h + z * q, the products rounded separately like the reference's two multiplies
      v[i].x = __fadd_rn(__fmul_rn(z[i].x, h[i].x), v[i].x); v[i].y = __fadd_rn(__fmul_rn(z[i].y, h[i].y), v[i].y);
      v[i].z = __fadd_rn(__fmul_rn(z[i].z, h[i].z), v[i].z); v[i].w = __fadd_rn(__fmul_rn(z[i].w, h[i].w), v[i].w);
    }
  }
  if (ep.res_f32) {
    float4 t[8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
      t[i] = (okm >> i) & 1 ? *reinterpret_cast<const float4*>(ep.res_f32 + (size_t)dr[i] * ep.res_f32_ld + col)
                            : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int i = 0; i < 8; ++i) { v[i].x += t[i].x; v[i].y += t[i].y; v[i].z += t[i].z; v[i].w += t[i].w; }
  }
  if (ep.res_a) {
    uint2 t[8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
      t[i] = (okm >> i) & 1 ? *reinterpret_cast<const uint2*>(ep.res_a + (size_t)dr[i] * ep.res_a_ld + col) : make_uint2(0u, 0u);
#pragma unroll
    for (int i = 0; i < 8; ++i) add_h4(v[i], t[i]);
  }
  if (ep.res_b) {
    uint2 t[8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
      t[i] = (okm >> i) & 1 ? *reinterpret_cast<const uint2*>(ep.res_b + (size_t)dr[i] * ep.res_b_ld + col) : make_uint2(0u, 0u);
#pragma unroll
    for (int i = 0; i < 8; ++i) add_h4(v[i], t[i]);
  }
  if (ep.out_f32) {
#pragma unroll
    for (int i = 0; i < 8; ++i)
      if ((okm >> i) & 1) *reinterpret_cast<float4*>(ep.out_f32 + (size_t)dr[i] * ep.out_f32_ld + col) = v[i];
  }
  if (ep.out_f16) {
#pragma unroll
    for (int i = 0; i < 8; ++i)
      if ((okm >> i) & 1)
        *reinterpret_cast<uint2*>(ep.out_f16 + (size_t)dr[i] * ep.out_f16_ld + col) =
            make_uint2(pack_half2(v[i].x, v[i].y), pack_half2(v[i].z, v[i].w));
  }
  if (ep.out_f16_relu) {
#pragma unroll
    for (int i = 0; i < 8; ++i)
      if ((okm >> i) & 1)
        *reinterpret_cast<uint2*>(ep.out_f16_relu + (size_t)dr[i] * ep.out_f16_relu_ld + col) =
            make_uint2(pack_half2(fmaxf(v[i].x, 0.f), fmaxf(v[i].y, 0.f)), pack_half2(fmaxf(v[i].z, 0.f), fmaxf(v[i].w, 0.f)));
  }
}

// Staging of the accumulator fragment of one warp (16 rows: r0 = 16 * (warp & 1) + lane / 4 and r0 + 8 of its 32-row slab)
// into the 32 x 128 B swizzled boxes of the warp pair: buffer q (= buf0 + q * stride) receives columns [cb + q * W, + W) of
// the slab, W = 32 fp32 (raw or scaled for the fp32 TMA store) or 64 fp16 (the fp16 TMA store, bias + activation applied).
// The 16-byte slot of column group g in row r is g ^ (r & 7): the 128-byte TMA swizzle of a 1024-aligned buffer.
// Register indices are compile-time (the column block is selected by predicate), so the accumulators stay in registers.
template <int BN, int MODE>  // MODE 0: raw fp32, 1: fp32 alpha * acc + bias, * gamma, 2: fp16 act(alpha * acc + bias)
__device__ __forceinline__ void stage_fragment(const float* d, int cb, uint32_t buf0, uint32_t stride, const GemmEpilogue& ep,
                                               int n0, int N, int warp, int lane) {
  constexpr int GROUPS = MODE == 2 ? 16 : 8;  // 8-column groups per call
  const int r0 = (warp & 1) * 16 + (lane >> 2), tq = lane & 3;
#pragma unroll
  for (int jg = 0; jg < BN / 8; ++jg) {
    const int j = jg - cb / 8;
    if (j < 0 || j >= GROUPS) continue;
    float x[4] = {d[jg * 4], d[jg * 4 + 1], d[jg * 4 + 2], d[jg * 4 + 3]};  // (r0, c), (r0, c + 1), (r0 + 8, c), (r0 + 8, c + 1)
    if (MODE != 0) {
      const int n = n0 + jg * 8 + tq * 2;
      float2 b = make_float2(0.f, 0.f), g = make_float2(1.f, 1.f);
      if (n < N) {
        if (ep.bias != nullptr) b = __ldg(reinterpret_cast<const float2*>(ep.bias + n));
        if (MODE == 1 && ep.gamma != nullptr) g = __ldg(reinterpret_cast<const float2*>(ep.gamma + n));
      }
      x[0] = fmaf(x[0], ep.alpha, b.x) * g.x; x[1] = fmaf(x[1], ep.alpha, b.y) * g.y;
      x[2] = fmaf(x[2], ep.alpha, b.x) * g.x; x[3] = fmaf(x[3], ep.alpha, b.y) * g.y;
      if (MODE == 2 && ep.act == 1) {
#pragma unroll
        for (int q = 0; q < 4; ++q) x[q] = gelu_erf(x[q]);
      } else if (MODE == 2 && ep.act == 2) {
#pragma unroll
        for (int q = 0; q < 4; ++q) x[q] = fmaxf(x[q], 0.f);
      }
    }
    const uint32_t buf = buf0 + (j / (GROUPS / 2)) * stride;
    const int jj = j % (GROUPS / 2);
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      const int row = r0 + hr * 8;
      if (MODE == 2) {
        const uint32_t a = buf + row * 128 + ((jj ^ (row & 7)) << 4) + tq * 4;
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(a), "r"(pack_half2(x[2 * hr], x[2 * hr + 1])) : "memory");
      } else {
        const int cc = jj * 8 + tq * 2;
        const uint32_t a = buf + row * 128 + ((((cc >> 2)) ^ (row & 7)) << 4) + (cc & 3) * 4;
        asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a), "f"(x[2 * hr]), "f"(x[2 * hr + 1]) : "memory");
      }
    }
  }
}

template <int BN, bool TMAST, bool TF32, bool XACC>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
               const __grid_constant__ CUtensorMap tmD, const __grid_constant__ GemmArgs args) {
  using Cfg = GemmCfg<BN, TMAST>;
  constexpr int STAGES = Cfg::STAGES;
  constexpr int BKE = TF32 ? 32 : 64;  // elements per 128-byte K block (fp32 containers for tf32, fp16 otherwise)
  extern __shared__ __align__(1024) uint8_t smem[];
  if ((smem_u32(smem) & 1023u) != 0) __trap();  // 128B-swizzle atoms are 1 KB
  uint8_t* sA = smem;
  uint8_t* sB = smem + STAGES * Cfg::A_BYTES;
  float* stg_all = reinterpret_cast<float*>(smem + STAGES * Cfg::STAGE_BYTES);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * Cfg::STAGE_BYTES + Cfg::STG_BYTES);
  uint64_t* full = bars;
  uint64_t* empty = bars + STAGES;

  pdl_launch_dependents();  // the next kernel may be scheduled behind this one (see common.cuh)
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = threadIdx.x >> 7;
  const int M_run = args.ep.m_dev ? min(args.M, (*args.ep.m_dev + GEMM_BM - 1) / GEMM_BM * GEMM_BM) : args.M;  // see GemmEpilogue::m_dev
  const int tiles_m = (M_run + GEMM_BM - 1) / GEMM_BM;
  const int tiles_n = (args.N + BN - 1) / BN;
  const int num_tiles = tiles_m * tiles_n;
  const int num_kb = args.taps * args.kchunks;
  auto tile_mn = [&](int tile, int* tm, int* tn) {
    *tm = args.raster_n ? tile / tiles_n : tile % tiles_m;
    *tn = args.raster_n ? tile % tiles_n : tile / tiles_m;
  };

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmA);
    prefetch_tmap(&tmB);
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 2); }  // empty: one arrival per consumer warpgroup
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();  // barriers and descriptors are set up; from here on the predecessor's results are read

  if (wg == 2) {
    // ------------------------------------------------------------------ TMA producer
    setmaxnreg_dec<40>();
    if (threadIdx.x == 256) {
      int stage = 0; uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        int tm, tn;
        tile_mn(tile, &tm, &tn);
        const int m0 = tm * GEMM_BM, n0 = tn * BN;
        int tap = 0, chunk = 0;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&empty[stage], phase ^ 1);
          mbar_arrive_expect_tx(&full[stage], Cfg::STAGE_BYTES);
          tma_load_2d(sA + stage * Cfg::A_BYTES, &tmA, &full[stage], args.tap_acol[tap] + chunk * BKE, m0 + args.tap_off[tap]);
          tma_load_2d(sB + stage * Cfg::B_BYTES, &tmB, &full[stage], kb * BKE, n0);
          if (++chunk == args.kchunks) { chunk = 0; ++tap; }
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ------------------------------------------------------------------ consumers: MMA + epilogue of 64 rows each
    setmaxnreg_inc<232>();
    const int slab = warp >> 1;    // 32-row slab of the tile this warp pair stores (0..3)
    const int half = warp & 1;     // which 32-column chunk of a 64-column block this warp stores
    const int pair_bar = 1 + slab;
    const GemmEpilogue& ep = args.ep;
    const uint32_t stg = smem_u32(stg_all) + warp * Cfg::STG_WARP;
    const uint32_t stg_pair = smem_u32(stg_all) + (warp & ~1) * Cfg::STG_WARP;
    uint32_t st_cnt = 0;  // TMAST: boxes stored so far by this warp (staging buffer parity)
    const int cg = lane & 7;     // coalesced phase: which 4-column group of the 32-column chunk
    const int rsub = lane >> 3;  // coalesced phase: row offset inside a 4-row step
    float acc[BN / 2];
    float run[XACC ? BN / 2 : 1];
    int stage = 0; uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      int tm, tn;
      tile_mn(tile, &tm, &tn);
      const int m0 = tm * GEMM_BM, n0 = tn * BN;
      // ---- mainloop
      if (XACC) {
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) run[i] = 0.f;
      }
      int prev_stage = -1;  // stage read by the wgmma group still in flight
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&full[stage], phase);
        const uint64_t adesc = make_wgmma_desc(smem_u32(sA + stage * Cfg::A_BYTES + wg * 64 * 128));
        const uint64_t bdesc = make_wgmma_desc(smem_u32(sB + stage * Cfg::B_BYTES));
        // External accumulation (XACC): the tensor core adds into its fp32 accumulator by TRUNCATING the aligned addend, a
        // bias that grows with the length of the chain.  Here a chain is only `acc_group` K blocks long; every finished
        // partial sum is added to register-resident running sums with round-to-nearest FADDs.
        const bool first = XACC ? (kb % args.acc_group) == 0 : kb == 0;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < GEMM_BK / 16; ++k) {
          // advance 32 B along K inside the 128 B swizzled row: +2 in the (addr >> 4) field
          if (TF32) Wgmma<BN>::tf32(acc, adesc + 2 * k, bdesc + 2 * k, (first && k == 0) ? 0 : 1);
          else Wgmma<BN>::f16(acc, adesc + 2 * k, bdesc + 2 * k, (first && k == 0) ? 0 : 1);
        }
        wgmma_commit();
        // one wgmma group stays in flight while the next stage is waited for: a stage is released when the group that
        // read it has retired, one K block later; the chain is drained at the end of a tile (and at the end of an XACC
        // group, whose partial sum is read here)
        if (XACC && (kb % args.acc_group) == args.acc_group - 1 && kb != num_kb - 1) {
          wgmma_wait<0>();
          if ((threadIdx.x & 127) == 0) {
            if (prev_stage >= 0) mbar_arrive(&empty[prev_stage]);
            mbar_arrive(&empty[stage]);
          }
          prev_stage = -1;
#pragma unroll
          for (int i = 0; i < BN / 2; ++i) run[i] += acc[i];
        } else {
          wgmma_wait<1>();
          if ((threadIdx.x & 127) == 0 && prev_stage >= 0) mbar_arrive(&empty[prev_stage]);
          prev_stage = stage;
        }
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      if ((threadIdx.x & 127) == 0 && prev_stage >= 0) mbar_arrive(&empty[prev_stage]);
      if (XACC) {
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) run[i] += acc[i];
      }
      const float* fin = XACC ? run : acc;

      if (TMAST) {
        // ---- TMA-store path: scaled (+ bias, LayerScale / activation) values straight into the swizzled boxes of the warp
        // pair, then one cp.async.bulk.tensor store (or reduce-add) per box by lane 0; two boxes per warp so that the store
        // of one block reads shared memory while the next is being staged
        const bool f16o = ep.out_f16 != nullptr;
        const int CB = f16o ? 128 : 64;  // columns of one pair iteration: two boxes of 64 fp16 / 32 fp32 columns
#pragma unroll 1
        for (int cb = 0; cb < BN && n0 + cb < args.N; cb += CB) {
          const uint32_t par = (st_cnt & 1) * 4096;
          if (st_cnt >= 2) { if (lane == 0) tma_store_wait_read<1>(); __syncwarp(); }
          named_bar_sync(pair_bar, 64);  // both boxes of this parity are free
          if (f16o) stage_fragment<BN, 2>(fin, cb, stg_pair + par, Cfg::STG_WARP, ep, n0, args.N, warp, lane);
          else stage_fragment<BN, 1>(fin, cb, stg_pair + par, Cfg::STG_WARP, ep, n0, args.N, warp, lane);
          fence_proxy_async_smem();
          named_bar_sync(pair_bar, 64);
          if (lane == 0) {
            const int c = n0 + cb + half * (CB / 2);
            if (cb + half * (CB / 2) < BN && c < args.N) {
              if (ep.tma_reduce)
                asm volatile("cp.reduce.async.bulk.tensor.2d.global.shared::cta.add.tile.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                                 reinterpret_cast<uint64_t>(&tmD)),
                             "r"(stg + par), "r"(c), "r"(m0 + slab * 32)
                             : "memory");
              else
                asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                                 reinterpret_cast<uint64_t>(&tmD)),
                             "r"(stg + par), "r"(c), "r"(m0 + slab * 32)
                             : "memory");
            }
            tma_store_commit();  // an empty group when this warp's box lies beyond N: keeps the parity count of both warps equal
          }
          ++st_cnt;
        }
        continue;
      }

      // ---- row mapping of the 32 output rows of this warp pair's slab (lane == row inside the slab)
      int m = 0, valid = 0, drow = 0;
      int ty = 0, tx = 0, img_base = 0;  // token coordinates / image base row for ROW_SHUFFLE
      const int out_ld = ep.out_lead < 0 ? ep.out_pad : ep.out_lead;  // leading border of the destination map
      int dr8[8], ty8[8], tx8[8], ib8[8];
      uint32_t okrows = 0;
      {
        m = m0 + slab * 32 + lane;
        valid = m < args.M;
        drow = m;
        if (ep.row_map == ROW_PADDED || ep.row_map == ROW_PAD2TOK) {
          int img = 0, r = m;
          if (ep.img_rows > 0) { img = m / ep.img_rows; r = m - img * ep.img_rows; }
          const int y = r / ep.in_w, x = r - y * ep.in_w;
          const int pd = ep.pad, ld = ep.lead < 0 ? ep.pad : ep.lead;
          valid = valid && y >= ld && y < ep.in_h - pd && x >= ld && x < ep.in_w - pd;
          if (ep.row_map == ROW_PAD2TOK) {
            const int ho = (ep.in_h - pd - ld + ep.sub - 1) / ep.sub, wo = (ep.in_w - pd - ld + ep.sub - 1) / ep.sub;
            valid = valid && ((y - ld) % ep.sub == 0) && ((x - ld) % ep.sub == 0);
            drow = img * (ep.out_img_rows > 0 ? ep.out_img_rows : ho * wo) + ((y - ld) / ep.sub) * wo + (x - ld) / ep.sub;
          } else if (ep.sub > 1 || ep.out_wp > 0) {
            // destination geometry differs from the source one (stride-2 sub-sampling and / or another border width)
            valid = valid && ((y - ld) % ep.sub == 0) && ((x - ld) % ep.sub == 0);
            drow = img * ep.out_img_rows + ((y - ld) / ep.sub + out_ld) * ep.out_wp + (x - ld) / ep.sub + out_ld;
          }
        } else if (ep.row_map == ROW_TOKSKIP) {
          drow = m + m / ep.in_w + 1;
        } else if (ep.row_map == ROW_TOK2PAD || ep.row_map == ROW_SHUFFLE) {
          const int per = ep.in_w * ep.in_h;
          const int img = m / per, r = m - img * per;
          ty = r / ep.in_w; tx = r - ty * ep.in_w;
          img_base = img * ep.out_img_rows;
          drow = img_base + (ty + out_ld) * ep.out_wp + tx + out_ld;
        }
        // row mapping of the 8 rows this lane stores in the coalesced phase
#pragma unroll
        for (int rr = 0; rr < 8; ++rr) {
          const int row = rr * 4 + rsub;
          okrows |= (__shfl_sync(0xffffffffu, valid, row) ? 1u : 0u) << rr;
          dr8[rr] = __shfl_sync(0xffffffffu, drow, row);
          if (ep.row_map == ROW_SHUFFLE) {
            ty8[rr] = __shfl_sync(0xffffffffu, ty, row);
            tx8[rr] = __shfl_sync(0xffffffffu, tx, row);
            ib8[rr] = __shfl_sync(0xffffffffu, img_base, row);
          }
        }
      }
#pragma unroll 1
      for (int cb = 0; cb < BN && n0 + cb < args.N; cb += 64) {
        named_bar_sync(pair_bar, 64);  // the partner has finished reading its buffer
        stage_fragment<BN, 0>(fin, cb, stg_pair, Cfg::STG_WARP, ep, n0, args.N, warp, lane);
        named_bar_sync(pair_bar, 64);
        const int c0 = cb + half * 32;
        if (c0 >= BN || n0 + c0 >= args.N) continue;  // warp-uniform
        if (ep.head_w != nullptr) {
          // fused DPT output head (N == 32): the lane's own row, all 32 columns
          if (valid) {
            float acc_h = ep.head_b;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const float4 q = lds128(stg + lane * 128 + ((j ^ (lane & 7)) << 4));
              const float r4[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
              for (int t = 0; t < 4; ++t) acc_h = fmaf(fmaxf(r4[t] + __ldg(ep.bias + 4 * j + t), 0.f), __ldg(ep.head_w + 4 * j + t), acc_h);
            }
            int img = 0, rpix = m;
            if (ep.img_rows > 0) { img = m / ep.img_rows; rpix = m - img * ep.img_rows; }
            const int y = rpix / ep.in_w, x = rpix - y * ep.in_w, pd = ep.pad;
            const size_t pix = ((size_t)img * (ep.in_h - 2 * pd) + (y - pd)) * (ep.in_w - 2 * pd) + (x - pd);
            ep.head_out[pix] = fmaxf(acc_h, 0.f);
            if (ep.out_f16) {  // also keep the 32 ReLU'd activations (the out_conv hook of the metric head), dense rows
              uint4* dst = reinterpret_cast<uint4*>(ep.out_f16 + pix * ep.out_f16_ld);
#pragma unroll
              for (int j = 0; j < 4; ++j) {
                const float4 a = lds128(stg + lane * 128 + (((2 * j) ^ (lane & 7)) << 4));
                const float4 b = lds128(stg + lane * 128 + (((2 * j + 1) ^ (lane & 7)) << 4));
                const float* bs = ep.bias + 8 * j;
                dst[j] = make_uint4(pack_half2(fmaxf(a.x + __ldg(bs), 0.f), fmaxf(a.y + __ldg(bs + 1), 0.f)),
                                    pack_half2(fmaxf(a.z + __ldg(bs + 2), 0.f), fmaxf(a.w + __ldg(bs + 3), 0.f)),
                                    pack_half2(fmaxf(b.x + __ldg(bs + 4), 0.f), fmaxf(b.y + __ldg(bs + 5), 0.f)),
                                    pack_half2(fmaxf(b.z + __ldg(bs + 6), 0.f), fmaxf(b.w + __ldg(bs + 7), 0.f)));
              }
            }
          }
          continue;
        }
        // ---- coalesced phase: 8 lanes x 4 columns cover one row's 32 columns; 4 rows per step
        const int n = n0 + c0 + cg * 4;
        const bool ncol_ok = n < args.N;
        float4 bias4 = make_float4(0.f, 0.f, 0.f, 0.f), gamma4 = make_float4(1.f, 1.f, 1.f, 1.f);
        if (ncol_ok && ep.bias) bias4 = *reinterpret_cast<const float4*>(ep.bias + n);
        if (ncol_ok && ep.gamma) gamma4 = *reinterpret_cast<const float4*>(ep.gamma + n);
        float4 v[8];
#pragma unroll
        for (int rr = 0; rr < 8; ++rr) {
          const int row = rr * 4 + rsub;
          v[rr] = lds128(stg + row * 128 + ((cg ^ (row & 7)) << 4));
        }
        int col = n;
        if (ep.row_map == ROW_SHUFFLE) {
          const int q = n / ep.shuf_cout;
          col = n - q * ep.shuf_cout;
          const int sdy = q / ep.shuf_s, sdx = q - sdy * ep.shuf_s;
          int drs[8];
#pragma unroll
          for (int rr = 0; rr < 8; ++rr)
            drs[rr] = ib8[rr] + (ty8[rr] * ep.shuf_s + sdy + out_ld) * ep.out_wp + tx8[rr] * ep.shuf_s + sdx + out_ld;
          epilogue_rows8<!TF32 && !XACC>(ep, v, drs, ncol_ok ? okrows : 0u, bias4, gamma4, col);
        } else {
          epilogue_rows8<!TF32 && !XACC>(ep, v, dr8, ncol_ok ? okrows : 0u, bias4, gamma4, col);
        }
        if (ep.stat_part != nullptr) {
          float4 sm = make_float4(0.f, 0.f, 0.f, 0.f), sq = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
          for (int rr = 0; rr < 8; ++rr)
            if ((okrows >> rr) & 1) {
              sm.x += v[rr].x; sm.y += v[rr].y; sm.z += v[rr].z; sm.w += v[rr].w;
              sq.x = fmaf(v[rr].x, v[rr].x, sq.x); sq.y = fmaf(v[rr].y, v[rr].y, sq.y);
              sq.z = fmaf(v[rr].z, v[rr].z, sq.z); sq.w = fmaf(v[rr].w, v[rr].w, sq.w);
            }
#pragma unroll
          for (int o = 8; o <= 16; o <<= 1) {  // the 4 lanes that hold the same 4 columns (rows rsub, rsub + 4, ...)
            sm.x += __shfl_xor_sync(0xffffffffu, sm.x, o); sm.y += __shfl_xor_sync(0xffffffffu, sm.y, o);
            sm.z += __shfl_xor_sync(0xffffffffu, sm.z, o); sm.w += __shfl_xor_sync(0xffffffffu, sm.w, o);
            sq.x += __shfl_xor_sync(0xffffffffu, sq.x, o); sq.y += __shfl_xor_sync(0xffffffffu, sq.y, o);
            sq.z += __shfl_xor_sync(0xffffffffu, sq.z, o); sq.w += __shfl_xor_sync(0xffffffffu, sq.w, o);
          }
          if (rsub == 0 && ncol_ok) {
            const size_t sl = (size_t)(m0 + slab * 32) >> 5;
            *reinterpret_cast<float4*>(ep.stat_part + (sl * 2) * args.N + n) = sm;
            *reinterpret_cast<float4*>(ep.stat_part + (sl * 2 + 1) * args.N + n) = sq;
          }
        }
      }
    }
    if (TMAST && lane == 0) tma_store_wait_all();  // shared memory must outlive the last bulk stores
  }
}
#endif  // __CUDACC__

// Host-side prepared launch: tensor maps encoded once, replayed every frame (also inside CUDA graphs).
struct GemmLaunch {
  CUtensorMap tmA, tmB;
  CUtensorMap tmD;             // dense output, 32-row boxes (TMA-store epilogue only)
  bool tma_store = false;
  bool xacc = false;           // external fp32 accumulation (tf32x3 only): see GemmArgs::acc_group
  bool tf32 = false;           // tf32 operands (fp32 containers): the 3xTF32 "fp32-class" path of the mask band
  GemmArgs args;
  int bn = 128;
  int grid = 1;
  double flops = 0;  // algorithmic 2*M*N*K (excluding border/padding waste)
};

// A: fp16 [a_rows][a_cols] with pitch a_pitch (elements);  W: fp16 [w_rows >= round_up(N, bn)][taps*kchunks*64]
int gemm_prepare(GemmLaunch* out, const __half* A, long long a_rows, int a_cols, int a_pitch, const __half* W,
                 int w_rows, int M, int N, int taps, const int* tap_off, const GemmEpilogue& ep, int num_sms,
                 int force_bn = 0);
// 3xTF32: A = fp32 [a_rows][2 * C_half] holding [hi | lo] halves (hi = the top 19 bits of the value, lo = value - hi) of
// which the first C channels enter the product, W = fp32 [w_rows][taps * 3 * C] holding per tap [W_hi | W_hi | W_lo];
// D = sum_t (hi . W_hi + lo . W_hi + hi . W_lo): fp32-class products (the dropped lo . W_lo term is 2^-22 relative), fp32
// accumulate.  Same epilogues.  C, C_half multiples of 32.
int gemm_prepare_tf32x3(GemmLaunch* out, const float* A_split, long long a_rows, int C, int C_half, const float* W3, int w_rows,
                        int M, int N, int taps, const int* tap_off, const GemmEpilogue& ep, int num_sms, int force_bn = 0);
int gemm_run(const GemmLaunch& g, cudaStream_t stream);
int gemm_pick_bn(int M, int N, int num_sms);

}  // namespace prisma
