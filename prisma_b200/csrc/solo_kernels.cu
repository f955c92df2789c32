// prisma_b200 -- SOLOv2 (mask_mmdet band) kernels outside the wgmma GEMM core: test-pipeline pre-process, the
// pooling / resampling glue of ResNet + FPN + SOLOV2Head, GroupNorm, and the whole decode (candidate selection, mask
// statistics, Matrix NMS, the two chained bilinear resizes to the frame, the band's union mask).  Reference files are
// cited per kernel (paths relative to bands/mmdet/).  All HBM- or latency-bound; nothing here is a GEMM.
#include "solo_kernels.cuh"

#include <math.h>

namespace prisma {

// ------------------------------------------------------------------------------------------------
// Test pipeline (_base_/datasets/coco_instance.py:16-32): mmcv.imrescale = cv2.resize(INTER_LINEAR) on u8, then
// imnormalize (f32: subtract mean, multiply by 1/std), then zero pad to a multiple of 32.
// cv2's 8-bit bilinear (cv::resize INTER_LINEAR on CV_8U; IPP is not used for it) is fixed point: tap weights rounded
// to 1/2048, horizontal pass in int, vertical pass (((b0 * (S0 >> 4)) >> 16) + ((b1 * (S1 >> 4)) >> 16) + 2) >> 2.
// The two axes treat the image border differently: the horizontal tap table clamps the position AND zeroes the
// fraction outside [0, W-1] (resize.cpp: "if (sx < 0) fx = 0, sx = 0"), the vertical pass keeps the fraction and only
// clips the two row indices -- so in border rows both truncating products are applied to the same row.  Byte-equal to
// cv2 4.13 for up- and down-scaling (tests/test_mask_gpu.py, np.array_equal).
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void cv_linear_tap(int d, double scale, int ssize, bool clamp_fraction, int* s0, int* s1, int* a0,
                                              int* a1) {
  float f = (float)((d + 0.5) * scale - 0.5);
  int s = (int)floorf(f);
  f -= (float)s;
  if (clamp_fraction) {
    if (s < 0) { f = 0.f; s = 0; }
    if (s >= ssize - 1) { f = 0.f; s = ssize - 1; }
  }
  *s0 = min(max(s, 0), ssize - 1);
  *s1 = min(max(s + 1, 0), ssize - 1);
  *a0 = (int)(short)__float2int_rn((1.f - f) * 2048.f);
  *a1 = (int)(short)__float2int_rn(f * 2048.f);
}
__global__ void k_solo_preprocess(const uint8_t* __restrict__ img, int H, int W, int nh, int nw, int hp, int wp,
                                  double scale_x, double scale_y, float* __restrict__ out, uint8_t* __restrict__ resized) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= wp) return;
  const float mean[3] = {123.675f, 116.28f, 103.53f};
  const float stdinv[3] = {(float)(1.0 / (double)58.395f), (float)(1.0 / (double)57.12f), (float)(1.0 / (double)57.375f)};
  if (x >= nw || y >= nh) {
#pragma unroll
    for (int c = 0; c < 3; ++c) out[((size_t)c * hp + y) * wp + x] = 0.f;
    return;
  }
  int sx, sx1, ax0, ax1, sy, sy1, by0, by1;
  cv_linear_tap(x, scale_x, W, true, &sx, &sx1, &ax0, &ax1);
  cv_linear_tap(y, scale_y, H, false, &sy, &sy1, &by0, &by1);
  const uint8_t* r0 = img + (size_t)sy * W * 3;
  const uint8_t* r1 = img + (size_t)sy1 * W * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const int S0 = r0[sx * 3 + c] * ax0 + r0[sx1 * 3 + c] * ax1;
    const int S1 = r1[sx * 3 + c] * ax0 + r1[sx1 * 3 + c] * ax1;
    const int v = (((by0 * (S0 >> 4)) >> 16) + ((by1 * (S1 >> 4)) >> 16) + 2) >> 2;
    const uint8_t u = (uint8_t)min(max(v, 0), 255);
    if (resized) resized[((size_t)y * nw + x) * 3 + c] = u;
    out[((size_t)c * hp + y) * wp + x] = __fmul_rn(__fsub_rn((float)u, mean[c]), stdinv[c]);
  }
}
int solo_preprocess(const uint8_t* rgb, int H, int W, int nh, int nw, int hp, int wp, float* out_chw, uint8_t* resized_u8,
                    cudaStream_t s) {
  dim3 grid(ceil_div(wp, 128), hp);
  k_solo_preprocess<<<grid, 128, 0, s>>>(rgb, H, W, nh, nw, hp, wp, 1.0 / ((double)nw / W), 1.0 / ((double)nh / H), out_chw,
                                         resized_u8);
  PRISMA_CUDA_OK(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------------------
// Zero-bordered NHWC fp16 maps (border 1), one image.  All kernels below index pixel (y, x) at row (y+1)*(W+2) + x+1.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ size_t prow(int y, int x, int W) { return (size_t)(y + 1) * (W + 2) + (x + 1); }

// nn.MaxPool2d(3, 2, 1) after the stem ReLU (models/backbones/resnet.py:608,639): inputs are >= 0, so the zero border
// plays the role of the -inf padding.
__global__ void k_maxpool3s2(const __half* __restrict__ in, int H, int W, int C, __half* __restrict__ out, int Ho, int Wo) {
  const int cv = C / 8;
  const long long total = (long long)Ho * Wo * cv;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c8 = (int)(i % cv);
    const int ox = (int)((i / cv) % Wo), oy = (int)(i / ((long long)cv * Wo));
    __half2 m[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) m[k] = __float2half2_rn(0.f);
#pragma unroll
    for (int dy = 0; dy < 3; ++dy)
#pragma unroll
      for (int dx = 0; dx < 3; ++dx) {
        const int py = 2 * oy + dy, px = 2 * ox + dx;  // padded coordinates of the input
        if (py > H + 1 || px > W + 1) continue;
        const uint4 v = *reinterpret_cast<const uint4*>(in + ((size_t)py * (W + 2) + px) * C + c8 * 8);
        const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
        for (int k = 0; k < 4; ++k) m[k] = __hmax2(m[k], h[k]);
      }
    *reinterpret_cast<uint4*>(out + prow(oy, ox, Wo) * C + c8 * 8) = *reinterpret_cast<uint4*>(m);
  }
}
int maxpool3s2_f16(const __half* in, int H, int W, int C, __half* out, int Ho, int Wo, cudaStream_t s) {
  k_maxpool3s2<<<device_sm_count() * 8, 256, 0, s>>>(in, H, W, C, out, Ho, Wo);
  PRISMA_CUDA_OK(cudaGetLastError());
  return 0;
}

// FPN top-down path (models/necks/fpn.py:166-177): fine += F.interpolate(coarse, size=fine.shape, mode="nearest");
// torch nearest: src = min(floor(dst * in/out), in - 1) with a float scale.
__global__ void k_nearest_add(__half* __restrict__ fine, int Hf, int Wf, const __half* __restrict__ coarse, int Hc, int Wc, int C,
                              float sy, float sx) {
  const int cv = C / 8;
  const long long total = (long long)Hf * Wf * cv;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c8 = (int)(i % cv);
    const int x = (int)((i / cv) % Wf), y = (int)(i / ((long long)cv * Wf));
    const int ys = min((int)floorf(y * sy), Hc - 1), xs = min((int)floorf(x * sx), Wc - 1);
    uint4 a = *reinterpret_cast<uint4*>(fine + prow(y, x, Wf) * C + c8 * 8);
    const uint4 b = *reinterpret_cast<const uint4*>(coarse + prow(ys, xs, Wc) * C + c8 * 8);
    __half2* ah = reinterpret_cast<__half2*>(&a);
    const __half2* bh = reinterpret_cast<const __half2*>(&b);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 fa = __half22float2(ah[k]), fb = __half22float2(bh[k]);
      ah[k] = __floats2half2_rn(fa.x + fb.x, fa.y + fb.y);
    }
    *reinterpret_cast<uint4*>(fine + prow(y, x, Wf) * C + c8 * 8) = a;
  }
}
int nearest_add_f16(__half* fine, int Hf, int Wf, const __half* coarse, int Hc, int Wc, int C, cudaStream_t s) {
  k_nearest_add<<<device_sm_count() * 4, 256, 0, s>>>(fine, Hf, Wf, coarse, Hc, Wc, C, (float)Hc / (float)Hf, (float)Wc / (float)Wf);
  PRISMA_CUDA_OK(cudaGetLastError());
  return 0;
}

// extra FPN level: F.max_pool2d(x, 1, stride=2) = x[::2, ::2] (fpn.py:188)
__global__ void k_subsample2(const __half* __restrict__ in, int H, int W, int C, __half* __restrict__ out, int Ho, int Wo) {
  const int cv = C / 8;
  const long long total = (long long)Ho * Wo * cv;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c8 = (int)(i % cv);
    const int x = (int)((i / cv) % Wo), y = (int)(i / ((long long)cv * Wo));
    *reinterpret_cast<uint4*>(out + prow(y, x, Wo) * C + c8 * 8) =
        *reinterpret_cast<const uint4*>(in + prow(2 * y, 2 * x, W) * C + c8 * 8);
  }
}
int subsample2_f16(const __half* in, int H, int W, int C, __half* out, int Ho, int Wo, cudaStream_t s) {
  k_subsample2<<<64, 256, 0, s>>>(in, H, W, C, out, Ho, Wo);
  PRISMA_CUDA_OK(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------------------
// GroupNorm(32, C, eps 1e-5) + ReLU of a ConvModule (mmcv ConvModule with norm_cfg=dict(type='GN', num_groups=32)).
// x: dense fp32 [HW][C] (conv output).  Deterministic: fixed row chunks -> per-channel partial (sum, sumsq) -> one block
// combines chunks and the channels of a group in a fixed order (double) -> per-channel (mean_g, rstd_g).
// ------------------------------------------------------------------------------------------------
constexpr int GN_CHUNK_ROWS = 256;
int gn_partial_floats(int HW, int C) { return ceil_div(HW, GN_CHUNK_ROWS) * C * 2; }

__global__ void k_gn_partial(const float* __restrict__ x, int HW, int C, float* __restrict__ part) {
  const int chunk = blockIdx.x, r0 = chunk * GN_CHUNK_ROWS, r1 = min(r0 + GN_CHUNK_ROWS, HW);
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float s = 0.f, q = 0.f;
    for (int r = r0; r < r1; ++r) { const float v = x[(size_t)r * C + c]; s += v; q = fmaf(v, v, q); }
    part[((size_t)chunk * C + c) * 2] = s;
    part[((size_t)chunk * C + c) * 2 + 1] = q;
  }
}
__global__ void k_gn_final(const float* __restrict__ part, int nchunks, int HW, int C, int groups, float* __restrict__ stats) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= groups) return;
  const int cpg = C / groups;
  double s = 0.0, q = 0.0;
  for (int k = 0; k < nchunks; ++k)
    for (int c = g * cpg; c < (g + 1) * cpg; ++c) { s += part[((size_t)k * C + c) * 2]; q += part[((size_t)k * C + c) * 2 + 1]; }
  const double n = (double)HW * cpg, mean = s / n, var = fmax(q / n - mean * mean, 0.0);
  const float rstd = (float)(1.0 / sqrt(var + 1e-5));
  for (int c = g * cpg; c < (g + 1) * cpg; ++c) { stats[2 * c] = (float)mean; stats[2 * c + 1] = rstd; }
}
__global__ void k_gn_apply(const float* __restrict__ x, int H, int W, int C, const float* __restrict__ stats,
                           const float* __restrict__ gamma, const float* __restrict__ beta, __half* __restrict__ out_padded,
                           __half* __restrict__ out_dense) {
  const int cv = C / 4;
  const long long total = (long long)H * W * cv;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c4 = (int)(i % cv) * 4;
    const long long pix = i / cv;
    const int xx = (int)(pix % W), yy = (int)(pix / W);
    const float4 v = *reinterpret_cast<const float4*>(x + (size_t)pix * C + c4);
    const float in[4] = {v.x, v.y, v.z, v.w};
    float o[4];
#pragma unroll
    for (int k = 0; k < 4; ++k)
      o[k] = fmaxf(fmaf((in[k] - stats[2 * (c4 + k)]) * stats[2 * (c4 + k) + 1], gamma[c4 + k], beta[c4 + k]), 0.f);
    const uint2 pk = make_uint2(pack_half2(o[0], o[1]), pack_half2(o[2], o[3]));
    if (out_padded) *reinterpret_cast<uint2*>(out_padded + prow(yy, xx, W) * C + c4) = pk;
    if (out_dense) *reinterpret_cast<uint2*>(out_dense + (size_t)pix * C + c4) = pk;
  }
}
// per-channel (mean_g, rstd_g) of GroupNorm(groups) over a dense fp32 [HW][C] conv output (shared with solo_exact.cu)
int gn_stats(const float* x, int HW, int C, int groups, float* part, float* stats, cudaStream_t s) {
  const int nchunks = ceil_div(HW, GN_CHUNK_ROWS);
  k_gn_partial<<<nchunks, 256, 0, s>>>(x, HW, C, part);
  k_gn_final<<<1, 32, 0, s>>>(part, nchunks, HW, C, groups, stats);
  PRISMA_CUDA_OK(cudaGetLastError());
  return 0;
}
int groupnorm_relu_f16(const float* x, int H, int W, int C, int groups, const float* gamma, const float* beta, float* part,
                       float* stats, __half* out_padded, __half* out_dense, cudaStream_t s) {
  PRISMA_TRY(gn_stats(x, H * W, C, groups, part, stats, s));
  k_gn_apply<<<device_sm_count() * 4, 256, 0, s>>>(x, H, W, C, stats, gamma, beta, out_padded, out_dense);
  PRISMA_CUDA_OK(cudaGetLastError());
  return 0;
}

// Stacked-grid variant for the head towers: one block per (frame, group); deterministic (fixed per-thread strides, fixed
// smem tree).  x: dense fp32 [B][F*F][C]; valid pixels of frame b: y, x < S[b].
__global__ void k_gn_grid(const float* __restrict__ x, int F, GridSizes S, int C, int groups, const float* __restrict__ gamma,
                          const float* __restrict__ beta, __half* __restrict__ out) {
  const int b = blockIdx.y, g = blockIdx.x, Sb = S.s[b], cpg = C / groups, n = Sb * Sb * cpg;
  const float* xb = x + (size_t)b * F * F * C + g * cpg;
  __shared__ double sh_s[256], sh_q[256];
  double s = 0.0, q = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const int c = i % cpg, p = i / cpg, yy = p / Sb, xx = p - yy * Sb;
    const float v = xb[(size_t)(yy * F + xx) * C + c];
    s += v; q += (double)v * v;
  }
  sh_s[threadIdx.x] = s; sh_q[threadIdx.x] = q;
  __syncthreads();
  for (int o = blockDim.x >> 1; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) { sh_s[threadIdx.x] += sh_s[threadIdx.x + o]; sh_q[threadIdx.x] += sh_q[threadIdx.x + o]; }
    __syncthreads();
  }
  const double mean = sh_s[0] / n, var = fmax(sh_q[0] / n - mean * mean, 0.0);
  const float mu = (float)mean, rstd = (float)(1.0 / sqrt(var + 1e-5));
  __half* ob = out + (size_t)b * (F + 2) * (F + 2) * C + g * cpg;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const int c = i % cpg, p = i / cpg, yy = p / Sb, xx = p - yy * Sb;
    const float v = xb[(size_t)(yy * F + xx) * C + c];
    ob[prow(yy, xx, F) * C + c] = __float2half_rn(fmaxf(fmaf((v - mu) * rstd, gamma[g * cpg + c], beta[g * cpg + c]), 0.f));
  }
}
int groupnorm_relu_grid_f16(const float* x, int B, int F, GridSizes S, int C, int groups, const float* gamma, const float* beta,
                            __half* out_padded, cudaStream_t s) {
  k_gn_grid<<<dim3(groups, B), 256, 0, s>>>(x, F, S, C, groups, gamma, beta, out_padded);
  PRISMA_CUDA_OK(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------------------
// F.interpolate(mode="bilinear", align_corners=False) between zero-bordered NHWC fp16 maps (nn.Upsample x2 of the mask
// feature head solov2_head.py:101-121, resize_feats solo_head.py:133-153, the S x S grid resize solov2_head.py:266-270),
// optionally appending generate_coordinate (core/utils/misc.py:190-208) channels of the source grid.
// torch: src = max(scale * (dst + 0.5) - 0.5, 0), scale = in / out (float).
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float linspace_m1_1(int i, int n) {  // torch.linspace(-1, 1, n)[i], fp32, symmetric evaluation
  if (n == 1) return -1.f;
  const float step = 2.f / (float)(n - 1);
  return i < n / 2 ? -1.f + step * (float)i : 1.f - step * (float)(n - 1 - i);
}
__global__ void k_resize_bilinear(const __half* __restrict__ src, int Hs, int Ws, int Cs, __half* __restrict__ dst, int Hd, int Wd,
                                  int Cd, float sy, float sx, int coord, int accumulate, int Wdf) {
  const int cv = Cs / 8 + (coord ? 1 : 0);
  const long long total = (long long)Hd * Wd * cv;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c8 = (int)(i % cv);
    const int x = (int)((i / cv) % Wd), y = (int)(i / ((long long)cv * Wd));
    const float fy = fmaxf(sy * (y + 0.5f) - 0.5f, 0.f), fx = fmaxf(sx * (x + 0.5f) - 0.5f, 0.f);
    const int y0 = (int)fy, x0 = (int)fx;
    const int y1 = y0 + (y0 < Hs - 1 ? 1 : 0), x1 = x0 + (x0 < Ws - 1 ? 1 : 0);
    const float ly = fy - y0, lx = fx - x0, hy = 1.f - ly, hx = 1.f - lx;
    __half* d = dst + prow(y, x, Wdf) * Cd + c8 * 8;
    if (c8 * 8 >= Cs) {  // the two coordinate channels (+ six zero channels of the 8-vector)
      const float cx = hy * (hx * linspace_m1_1(x0, Ws) + lx * linspace_m1_1(x1, Ws)) + ly * (hx * linspace_m1_1(x0, Ws) + lx * linspace_m1_1(x1, Ws));
      const float cy = hy * (hx * linspace_m1_1(y0, Hs) + lx * linspace_m1_1(y0, Hs)) + ly * (hx * linspace_m1_1(y1, Hs) + lx * linspace_m1_1(y1, Hs));
      *reinterpret_cast<uint4*>(d) = make_uint4(pack_half2(cx, cy), 0u, 0u, 0u);
      continue;
    }
    const uint4 a = *reinterpret_cast<const uint4*>(src + prow(y0, x0, Ws) * Cs + c8 * 8);
    const uint4 b = *reinterpret_cast<const uint4*>(src + prow(y0, x1, Ws) * Cs + c8 * 8);
    const uint4 c = *reinterpret_cast<const uint4*>(src + prow(y1, x0, Ws) * Cs + c8 * 8);
    const uint4 e = *reinterpret_cast<const uint4*>(src + prow(y1, x1, Ws) * Cs + c8 * 8);
    const __half2 *ah = reinterpret_cast<const __half2*>(&a), *bh = reinterpret_cast<const __half2*>(&b);
    const __half2 *ch = reinterpret_cast<const __half2*>(&c), *eh = reinterpret_cast<const __half2*>(&e);
    uint4 o;
    if (accumulate) o = *reinterpret_cast<const uint4*>(d);
    __half2* oh = reinterpret_cast<__half2*>(&o);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 fa = __half22float2(ah[k]), fb = __half22float2(bh[k]), fc = __half22float2(ch[k]), fe = __half22float2(eh[k]);
      float vx = hy * (hx * fa.x + lx * fb.x) + ly * (hx * fc.x + lx * fe.x);
      float vy = hy * (hx * fa.y + lx * fb.y) + ly * (hx * fc.y + lx * fe.y);
      if (accumulate) { const float2 p = __half22float2(oh[k]); vx += p.x; vy += p.y; }
      oh[k] = __floats2half2_rn(vx, vy);
    }
    *reinterpret_cast<uint4*>(d) = o;
  }
}
int resize_bilinear_f16(const __half* src, int Hs, int Ws, int Csrc, __half* dst, int Hd, int Wd, int Cdst, int coord,
                        int accumulate, cudaStream_t s, int dst_frame_w) {
  k_resize_bilinear<<<device_sm_count() * 4, 256, 0, s>>>(src, Hs, Ws, Csrc, dst, Hd, Wd, Cdst, (float)Hs / (float)Hd, (float)Ws / (float)Wd,
                                           coord, accumulate, dst_frame_w > 0 ? dst_frame_w : Wd);
  PRISMA_CUDA_OK(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------------------
// Decode, step 1 (solov2_head.py:611-617,694-703): sigmoid, points NMS (2x2 max-pool, keep cells equal to their local
// maximum), score_thr -> candidate list.  cls_logits: dense fp32 [S*S][num_classes] of one level.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float sigmoid_ref(float x) { return 1.0f / (1.0f + expf(-x)); }
__global__ void k_solo_candidates(const float* __restrict__ logits, int S, int cell0, int NC, float thr, float stride,
                                  SoloCand* __restrict__ cand, int* __restrict__ count, int cap, int F) {
  const int total = S * S * NC;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int c = i % NC, cell = i / NC, y = cell / S, x = cell % S;
    const size_t row = (size_t)y * F + x;  // the logits live in an F-wide frame (F == S when not stacked)
    const float v = sigmoid_ref(logits[row * NC + c]);
    // local_max[y][x] of max_pool2d(k=2, stride 1, padding 1)[:-1, :-1] = max over (y-1..y, x-1..x)
    float m = v;
    if (x > 0) m = fmaxf(m, sigmoid_ref(logits[(row - 1) * NC + c]));
    if (y > 0) m = fmaxf(m, sigmoid_ref(logits[(row - F) * NC + c]));
    if (x > 0 && y > 0) m = fmaxf(m, sigmoid_ref(logits[(row - F - 1) * NC + c]));
    if (m == v && v > thr) {
      const int k = atomicAdd(count, 1);
      if (k < cap) { cand[k].score = v; cand[k].flat = (cell0 + cell) * NC + c; cand[k].area = 0.f; cand[k].stride = stride; }
    }
  }
}
int solo_candidates(const float* cls_logits, int S, int cell0, int num_classes, float score_thr, float stride, SoloCand* cand,
                    int* count, int cap, cudaStream_t s, int frame) {
  k_solo_candidates<<<64, 256, 0, s>>>(cls_logits, S, cell0, num_classes, score_thr, stride, cand, count, cap, frame > 0 ? frame : S);
  PRISMA_CUDA_OK(cudaGetLastError());
  return 0;
}

// one-block bitonic sort of up to SORT_CAP 64-bit keys (ascending); the low 32 bits carry the payload index
constexpr int SORT_CAP = 4096;
__device__ void bitonic_sort_block(unsigned long long* keys, int n_pow2) {
  for (int k = 2; k <= n_pow2; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      __syncthreads();
      for (int i = threadIdx.x; i < n_pow2; i += blockDim.x) {
        const int l = i ^ j;
        if (l > i) {
          const bool up = (i & k) == 0;
          const unsigned long long a = keys[i], b = keys[l];
          if ((a > b) == up) { keys[i] = b; keys[l] = a; }
        }
      }
    }
  __syncthreads();
}
// candidates into the reference's nonzero() order (ascending flat index): the order every later "stable" step refers to
__global__ void k_solo_sort_flat(const SoloCand* __restrict__ in, int* __restrict__ count, int cap, SoloCand* __restrict__ out) {
  __shared__ unsigned long long keys[SORT_CAP];
  const int n = min(*count, cap);
  for (int i = threadIdx.x; i < SORT_CAP; i += blockDim.x)
    keys[i] = i < n ? (((unsigned long long)(unsigned)in[i].flat << 32) | (unsigned)i) : ~0ull;
  bitonic_sort_block(keys, SORT_CAP);
  for (int i = threadIdx.x; i < n; i += blockDim.x) out[i] = in[(unsigned)(keys[i] & 0xffffffffu)];
  __syncthreads();
  if (threadIdx.x == 0) *count = n;  // clamp to the capacity
}
int solo_sort_candidates(const SoloCand* cand, int* count, int cap, SoloCand* sorted, cudaStream_t s) {
  PRISMA_CHECK(cap <= SORT_CAP, "solo: candidate capacity above the sort capacity");
  k_solo_sort_flat<<<1, 1024, 0, s>>>(cand, count, cap, sorted);
  PRISMA_CUDA_OK(cudaGetLastError());
  return 0;
}

// kernel_preds[inds[:, 0]] (solov2_head.py:703): gather the 256-vector of each candidate's cell as an fp16 GEMM operand row
__global__ void k_solo_gather(const SoloCand* __restrict__ cand, const int* __restrict__ count, int cap,
                              const float* const* __restrict__ lvl_kernels, const int* __restrict__ lvl_cell0, int levels, int NC,
                              int C, __half* __restrict__ out, const int* __restrict__ lvl_S, int F) {
  const int r = blockIdx.x;
  const int n = min(*count, cap);
  __half* o = out + (size_t)r * C;
  if (r >= n) {
    for (int c = threadIdx.x; c < C; c += blockDim.x) o[c] = __float2half_rn(0.f);
    return;
  }
  const int cell = cand[r].flat / NC;
  int lvl = 0;
  while (lvl + 1 < levels && cell >= lvl_cell0[lvl + 1]) ++lvl;
  int local = cell - lvl_cell0[lvl];
  if (lvl_S) { const int S = lvl_S[lvl]; local = (local / S) * F + local % S; }  // cell (y, x) inside an F-wide frame
  const float* k = lvl_kernels[lvl] + (size_t)local * C;
  for (int c = threadIdx.x; c < C; c += blockDim.x) o[c] = __float2half_rn(k[c]);
}
int solo_gather_kernels(const SoloCand* cand, const int* count, int cap, const float* const* lvl_kernels,
                        const int* lvl_cell0, int levels, int num_classes, int C, __half* out, cudaStream_t s,
                        const int* lvl_S, int frame) {
  k_solo_gather<<<cap, 64, 0, s>>>(cand, count, cap, lvl_kernels, lvl_cell0, levels, num_classes, C, out, lvl_S, frame);
  PRISMA_CUDA_OK(cudaGetLastError());
  return 0;
}

// masks = p > thr ; sum_masks ; maskness = sum(p * mask) / sum_masks ; score *= maskness (solov2_head.py:724-739)
__device__ __forceinline__ float mask_f(__half v) { return __half2float(v); }
__device__ __forceinline__ float mask_f(float v) { return v; }
template <typename T>
__global__ void k_solo_mask_stats(const T* __restrict__ masks, int HW, float thr, SoloCand* __restrict__ cand,
                                  const int* __restrict__ count, int cap) {
  const int r = blockIdx.x;
  if (r >= min(*count, cap)) return;
  const T* p = masks + (size_t)r * HW;
  float area = 0.f, wsum = 0.f;
  for (int i = threadIdx.x; i < HW; i += blockDim.x) {
    const float v = mask_f(p[i]);
    if (v > thr) { area += 1.f; wsum += v; }
  }
  __shared__ float sa[32], sw[32];
  area = warp_sum(area); wsum = warp_sum(wsum);
  if ((threadIdx.x & 31) == 0) { sa[threadIdx.x >> 5] = area; sw[threadIdx.x >> 5] = wsum; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float a = 0.f, w = 0.f;
    for (int k = 0; k < (int)(blockDim.x >> 5); ++k) { a += sa[k]; w += sw[k]; }
    cand[r].area = a;
    cand[r].score = a > 0.f ? cand[r].score * (w / a) : 0.f;
  }
}
int solo_mask_stats(const __half* masks, int HW, float mask_thr, SoloCand* cand, const int* count, int cap,
                    cudaStream_t s) {
  k_solo_mask_stats<__half><<<cap, 256, 0, s>>>(masks, HW, mask_thr, cand, count, cap);
  PRISMA_CUDA_OK(cudaGetLastError());
  return 0;
}
int solo_mask_stats(const float* masks, int HW, float mask_thr, SoloCand* cand, const int* count, int cap, cudaStream_t s) {
  k_solo_mask_stats<float><<<cap, 256, 0, s>>>(masks, HW, mask_thr, cand, count, cap);
  PRISMA_CUDA_OK(cudaGetLastError());
  return 0;
}

// keep = sum_masks > strides, then torch.sort(scores, descending) and the first nms_pre (matrix_nms.py:56-63)
__global__ void k_solo_rank(const SoloCand* __restrict__ cand, const int* __restrict__ count, int cap, int nms_pre,
                            int* __restrict__ top, int* __restrict__ n_top) {
  __shared__ unsigned long long keys[SORT_CAP];
  __shared__ int valid;
  if (threadIdx.x == 0) valid = 0;
  __syncthreads();
  const int n = min(*count, cap);
  for (int i = threadIdx.x; i < SORT_CAP; i += blockDim.x) {
    unsigned long long k = ~0ull;
    if (i < n && cand[i].area > cand[i].stride) {
      k = ((unsigned long long)(0xffffffffu - __float_as_uint(cand[i].score)) << 32) | (unsigned)i;
      atomicAdd(&valid, 1);
    }
    keys[i] = k;
  }
  bitonic_sort_block(keys, SORT_CAP);
  const int m = min(valid, nms_pre);
  for (int i = threadIdx.x; i < nms_pre; i += blockDim.x) top[i] = i < m ? (int)(keys[i] & 0xffffffffu) : -1;
  if (threadIdx.x == 0) *n_top = m;
}
int solo_rank(const SoloCand* cand, const int* count, int cap, int nms_pre, int* top, int* n_top,
              cudaStream_t s) {
  k_solo_rank<<<1, 1024, 0, s>>>(cand, count, cap, nms_pre, top, n_top);
  PRISMA_CUDA_OK(cudaGetLastError());
  return 0;
}

// binary masks of the ranked candidates as an fp16 0/1 matrix [nms_pre_pad][HW]: the operand of inter = M M^T
template <typename T>
__global__ void k_solo_binarize(const T* __restrict__ masks, int HW, float thr, const int* __restrict__ top,
                                const int* __restrict__ n_top, __half* __restrict__ bin) {
  const int k = blockIdx.x;
  __half* o = bin + (size_t)k * HW;
  const int r = k < *n_top ? top[k] : -1;
  const __half one = __float2half_rn(1.f), zero = __float2half_rn(0.f);
  for (int i = threadIdx.x; i < HW; i += blockDim.x)
    o[i] = (r >= 0 && mask_f(masks[(size_t)r * HW + i]) > thr) ? one : zero;
}
int solo_binarize(const __half* masks, int HW, float mask_thr, const int* top, const int* n_top, int nms_pre, __half* bin,
                  cudaStream_t s) {
  k_solo_binarize<__half><<<nms_pre, 256, 0, s>>>(masks, HW, mask_thr, top, n_top, bin);
  PRISMA_CUDA_OK(cudaGetLastError());
  return 0;
}
int solo_binarize(const float* masks, int HW, float mask_thr, const int* top, const int* n_top, int nms_pre, __half* bin,
                  cudaStream_t s) {
  k_solo_binarize<float><<<nms_pre, 256, 0, s>>>(masks, HW, mask_thr, top, n_top, bin);
  PRISMA_CUDA_OK(cudaGetLastError());
  return 0;
}

// mask_matrix_nms, gaussian kernel (core/post_processing/matrix_nms.py:64-121).  One block, n <= 512.
constexpr int NMS_CAP = 512;
__global__ void k_solo_matrix_nms(const float* __restrict__ inter, int ld, const SoloCand* __restrict__ cand,
                                  const int* __restrict__ top, const int* __restrict__ n_top, int NC, float sigma, float filter_thr,
                                  int max_num, int* __restrict__ keep, float* __restrict__ keep_score, int* __restrict__ keep_label,
                                  int* __restrict__ n_keep) {
  __shared__ float area[NMS_CAP], comp[NMS_CAP], score[NMS_CAP];
  __shared__ int label[NMS_CAP];
  __shared__ unsigned long long keys[NMS_CAP];
  __shared__ int valid;
  const int n = *n_top;
  if (threadIdx.x == 0) valid = 0;
  for (int j = threadIdx.x; j < n; j += blockDim.x) {
    const SoloCand c = cand[top[j]];
    area[j] = c.area; label[j] = c.flat % NC; score[j] = c.score;
  }
  __syncthreads();
  auto iou = [&](int i, int j) -> float {  // decay_iou[i][j]: upper triangle, same label
    if (i >= j || label[i] != label[j]) return 0.f;
    const float in = inter[(size_t)i * ld + j];
    return in / (area[i] + area[j] - in);
  };
  for (int j = threadIdx.x; j < n; j += blockDim.x) {  // compensate_iou = column max
    float m = 0.f;
    for (int i = 0; i < j; ++i) m = fmaxf(m, iou(i, j));
    comp[j] = m;
  }
  __syncthreads();
  for (int j = threadIdx.x; j < NMS_CAP; j += blockDim.x) {
    unsigned long long key = ~0ull;
    if (j < n) {
      float coef = INFINITY;
      for (int i = 0; i < n; ++i) {
        const float d = iou(i, j);
        coef = fminf(coef, expf(-1.f * sigma * (d * d)) / expf(-1.f * sigma * (comp[i] * comp[i])));
      }
      const float sc = score[j] * coef;
      score[j] = sc;
      if (sc >= filter_thr) { key = ((unsigned long long)(0xffffffffu - __float_as_uint(sc)) << 32) | (unsigned)j; atomicAdd(&valid, 1); }
    }
    keys[j] = key;
  }
  bitonic_sort_block(keys, NMS_CAP);
  const int m = min(valid, max_num);
  for (int i = threadIdx.x; i < max_num; i += blockDim.x) {
    if (i < m) {
      const int j = (int)(keys[i] & 0xffffffffu);
      keep[i] = top[j]; keep_score[i] = score[j]; keep_label[i] = label[j];
    } else { keep[i] = -1; keep_score[i] = 0.f; keep_label[i] = -1; }
  }
  if (threadIdx.x == 0) *n_keep = m;
}
int solo_matrix_nms(const float* inter, int ld, const SoloCand* cand, const int* top, const int* n_top, int num_classes,
                    float sigma, float filter_thr, int max_num, int* keep, float* keep_score, int* keep_label, int* n_keep,
                    cudaStream_t s) {
  k_solo_matrix_nms<<<1, 512, 0, s>>>(inter, ld, cand, top, n_top, num_classes, sigma, filter_thr, max_num, keep, keep_score,
                                      keep_label, n_keep);
  PRISMA_CUDA_OK(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------------------
// Final masks (solov2_head.py:751-762): interpolate the kept mask_preds to (4 fh, 4 fw), crop to img_shape, interpolate to
// ori_shape, threshold -- evaluated per output pixel as two nested bilinear taps -- and the band's frame
// (bands/mask_mmdet.py:43-61,134-146): 255 * (number of instances of the 11 classes above the confidences) mod 256.
// ------------------------------------------------------------------------------------------------
template <typename T>
__device__ __forceinline__ float up4_at(const T* __restrict__ p, int fh, int fw, int yy, int xx) {
  const float fy = fmaxf(0.25f * (yy + 0.5f) - 0.5f, 0.f), fx = fmaxf(0.25f * (xx + 0.5f) - 0.5f, 0.f);
  const int y0 = (int)fy, x0 = (int)fx;
  const int y1 = y0 + (y0 < fh - 1 ? 1 : 0), x1 = x0 + (x0 < fw - 1 ? 1 : 0);
  const float ly = fy - y0, lx = fx - x0, hy = 1.f - ly, hx = 1.f - lx;
  return hy * (hx * mask_f(p[y0 * fw + x0]) + lx * mask_f(p[y0 * fw + x1])) +
         ly * (hx * mask_f(p[y1 * fw + x0]) + lx * mask_f(p[y1 * fw + x1]));
}
__device__ __forceinline__ bool band_class(int l) { return l == 0 || (l >= 14 && l <= 23); }
template <typename T>
__global__ void k_solo_final(const T* __restrict__ masks, int fh, int fw, int h, int w, int H, int W, float thr,
                             const int* __restrict__ keep, const float* __restrict__ keep_score, const int* __restrict__ keep_label,
                             const int* __restrict__ n_keep, float confidence, float sy, float sx, uint8_t* __restrict__ inst,
                             uint8_t* __restrict__ uni) {
  const int n = *n_keep;
  const long long total = (long long)H * W;
  const int UH = 4 * fh, UW = 4 * fw;  // the up-sampled map before the [:h, :w] crop
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int Y = (int)(i / W), X = (int)(i - (long long)Y * W);
    const float fy = fmaxf(sy * (Y + 0.5f) - 0.5f, 0.f), fx = fmaxf(sx * (X + 0.5f) - 0.5f, 0.f);
    const int y0 = (int)fy, x0 = (int)fx;
    const int y1 = y0 + (y0 < h - 1 ? 1 : 0), x1 = x0 + (x0 < w - 1 ? 1 : 0);
    const float ly = fy - y0, lx = fx - x0, hy = 1.f - ly, hx = 1.f - lx;
    int count = 0;
    for (int k = 0; k < n; ++k) {
      const bool in_band = band_class(keep_label[k]) && keep_score[k] > 0.5f && keep_score[k] > confidence;
      if (!inst && !in_band) continue;
      const T* p = masks + (size_t)keep[k] * fh * fw;
      (void)UH; (void)UW;
      const float v = hy * (hx * up4_at(p, fh, fw, y0, x0) + lx * up4_at(p, fh, fw, y0, x1)) +
                      ly * (hx * up4_at(p, fh, fw, y1, x0) + lx * up4_at(p, fh, fw, y1, x1));
      const bool m = v > thr;
      if (inst) inst[(size_t)k * total + i] = m ? 1 : 0;
      if (m && in_band) ++count;
    }
    if (uni) uni[i] = (uint8_t)((255 * count) & 255);
  }
}
int solo_final_masks(const __half* masks, int fh, int fw, int h, int w, int H, int W, float mask_thr, const int* keep,
                     const float* keep_score, const int* keep_label, const int* n_keep, int max_num, float confidence,
                     uint8_t* inst_masks, uint8_t* union_mask, cudaStream_t s) {
  (void)max_num;
  k_solo_final<__half><<<device_sm_count() * 8, 256, 0, s>>>(masks, fh, fw, h, w, H, W, mask_thr, keep, keep_score, keep_label, n_keep, confidence,
                                              (float)h / (float)H, (float)w / (float)W, inst_masks, union_mask);
  PRISMA_CUDA_OK(cudaGetLastError());
  return 0;
}
int solo_final_masks(const float* masks, int fh, int fw, int h, int w, int H, int W, float mask_thr, const int* keep,
                     const float* keep_score, const int* keep_label, const int* n_keep, int max_num, float confidence,
                     uint8_t* inst_masks, uint8_t* union_mask, cudaStream_t s) {
  (void)max_num;
  k_solo_final<float><<<device_sm_count() * 8, 256, 0, s>>>(masks, fh, fw, h, w, H, W, mask_thr, keep, keep_score, keep_label, n_keep, confidence,
                                             (float)h / (float)H, (float)w / (float)W, inst_masks, union_mask);
  PRISMA_CUDA_OK(cudaGetLastError());
  return 0;
}


// ------------------------------------------------------------------------------------------------
// SDF of the union mask for --sdf (bands/mask_mmdet.py:64-69,150-152): snowy.generate_sdf(mask != 0) = udf(mask) - udf(~mask)
// with udf = exact Euclidean distance to the nearest set pixel (snowy: Felzenszwalb-Huttenlocher EDT, INF = 1e20, sqrt).
// Exact integer squared distances: pass 1 per column (nearest set pixel above / below), pass 2 per row by exhaustive
// minimisation over the row (W^2 H integer ops, ~1 ms at 1080p) -- same result as the lower-envelope algorithm.
// ------------------------------------------------------------------------------------------------
constexpr int SDF_INF = 1 << 28;
__global__ void k_sdf_columns(const uint8_t* __restrict__ mask, int H, int W, int* __restrict__ ga, int* __restrict__ gb) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= W) return;
  int da = SDF_INF, db = SDF_INF;  // distance to the last seen set (a) / unset (b) pixel above
  for (int y = 0; y < H; ++y) {
    const bool m = mask[(size_t)y * W + x] != 0;
    da = m ? 0 : (da >= SDF_INF ? SDF_INF : da + 1);
    db = !m ? 0 : (db >= SDF_INF ? SDF_INF : db + 1);
    ga[(size_t)y * W + x] = da; gb[(size_t)y * W + x] = db;
  }
  da = db = SDF_INF;
  for (int y = H - 1; y >= 0; --y) {
    const bool m = mask[(size_t)y * W + x] != 0;
    da = m ? 0 : (da >= SDF_INF ? SDF_INF : da + 1);
    db = !m ? 0 : (db >= SDF_INF ? SDF_INF : db + 1);
    ga[(size_t)y * W + x] = min(ga[(size_t)y * W + x], da);
    gb[(size_t)y * W + x] = min(gb[(size_t)y * W + x], db);
  }
}
__global__ void k_sdf_rows(const int* __restrict__ ga, const int* __restrict__ gb, int W, uint8_t* __restrict__ green) {
  extern __shared__ long long sq[];  // [2][W] squared column distances of this row
  const int y = blockIdx.x;
  long long* sa = sq; long long* sb = sq + W;
  for (int x = threadIdx.x; x < W; x += blockDim.x) {
    const int a = ga[(size_t)y * W + x], b = gb[(size_t)y * W + x];
    sa[x] = a >= SDF_INF ? -1 : (long long)a * a;
    sb[x] = b >= SDF_INF ? -1 : (long long)b * b;
  }
  __syncthreads();
  for (int x = threadIdx.x; x < W; x += blockDim.x) {
    long long da = -1, db = -1;
    for (int xp = 0; xp < W; ++xp) {
      const long long dx2 = (long long)(x - xp) * (x - xp);
      if (sa[xp] >= 0) { const long long v = sa[xp] + dx2; da = (da < 0 || v < da) ? v : da; }
      if (sb[xp] >= 0) { const long long v = sb[xp] + dx2; db = (db < 0 || v < db) ? v : db; }
    }
    // snowy: sqrt of the squared EDT, 1e20 where no set pixel exists at all
    const double ua = da < 0 ? 1e10 : sqrt((double)da), ub = db < 0 ? 1e10 : sqrt((double)db);
    double sdf = ua - ub;
    sdf = (sdf + 127.0) / 255.0;
    sdf = (sdf - 0.25) * 2.0;
    const double g = 1.0 - fmin(fmax(sdf, 0.0), 1.0);
    green[(size_t)y * W + x] = (uint8_t)(int)(g * 255.0);
  }
}
int mask_sdf_green(const uint8_t* mask, int H, int W, int* d_scratch, uint8_t* green, cudaStream_t s) {
  int* ga = d_scratch; int* gb = d_scratch + (size_t)H * W;
  k_sdf_columns<<<ceil_div(W, 128), 128, 0, s>>>(mask, H, W, ga, gb);
  k_sdf_rows<<<H, 256, 2 * W * sizeof(long long), s>>>(ga, gb, W, green);
  PRISMA_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace prisma
