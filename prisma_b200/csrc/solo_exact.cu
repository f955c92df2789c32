// prisma_b200 -- SOLOv2 "fp32-class" head: the kernels between the 3xTF32 GEMMs (gemm_prepare_tf32x3).
//
// north_star asks for bit-exact mask ids.  With single-pass fp16 (or tf32) operands the head's class scores move by ~2e-3
// and a third of the instance list changes against the fp32 reference; with fp32-class contractions the labels are equal,
// the scores agree to ~1e-6 and the masks differ in ~1e-7 of their bits (oracle emulation: 1 of 7.68 M on the pinned
// fixture).  So the mask band keeps every activation of the head in fp32 and feeds the tensor cores with [hi | lo] splits:
//
//   split map : zero-bordered NHWC, row = 2 C floats = [hi(C) | lo(C)], hi = the value with its low 13 mantissa bits
//               cleared (exactly a TF32 number), lo = value - hi (exact in fp32).  hi + lo reproduces the fp32 value, so the
//               map is a lossless fp32 activation AND the A operand of gemm_prepare_tf32x3.
//
// Kernels: loaders (dense fp32 / fp16 map -> split map), GroupNorm + ReLU apply (conv output -> split map or the
// [hi | hi | lo] "weight" layout of the dynamic convolution), bilinear resize (+ coordinate channels, + accumulate) between
// split maps, the candidate-kernel gather.  Statistics reuse k_gn_partial / k_gn_final.  Reference lines as in
// solo_kernels.cu.
#include <math.h>

#include "solo_kernels.cuh"

namespace prisma {

__device__ __forceinline__ size_t sprow(int y, int x, int W) { return (size_t)(y + 1) * (W + 2) + (x + 1); }
__device__ __forceinline__ float tf32_hi(float v) { return __uint_as_float(__float_as_uint(v) & 0xFFFFE000u); }
__device__ __forceinline__ void store_split4(float* row, int C, int c, const float4& v) {
  const float4 hi = make_float4(tf32_hi(v.x), tf32_hi(v.y), tf32_hi(v.z), tf32_hi(v.w));
  *reinterpret_cast<float4*>(row + c) = hi;
  *reinterpret_cast<float4*>(row + C + c) = make_float4(v.x - hi.x, v.y - hi.y, v.z - hi.z, v.w - hi.w);
}
__device__ __forceinline__ float4 load_split4(const float* row, int C, int c) {
  const float4 hi = *reinterpret_cast<const float4*>(row + c), lo = *reinterpret_cast<const float4*>(row + C + c);
  return make_float4(hi.x + lo.x, hi.y + lo.y, hi.z + lo.z, hi.w + lo.w);
}

// dense fp32 [H*W][Csrc] (NHWC) -> split map with Cdst >= Csrc channels (the extra channels stay zero)
__global__ void k_dense_to_split(const float* __restrict__ src, int H, int W, int Cs, float* __restrict__ dst, int Cd) {
  const int cv = Cs / 4;
  const long long total = (long long)H * W * cv;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % cv) * 4;
    const long long pix = i / cv;
    const int x = (int)(pix % W), y = (int)(pix / W);
    store_split4(dst + sprow(y, x, W) * 2 * Cd, Cd, c, *reinterpret_cast<const float4*>(src + (size_t)pix * Cs + c));
  }
}
int solo_dense_to_split(const float* src, int H, int W, int Csrc, float* dst, int Cdst, cudaStream_t s) {
  k_dense_to_split<<<device_sm_count() * 4, 256, 0, s>>>(src, H, W, Csrc, dst, Cdst);
  PRISMA_CUDA_OK(cudaGetLastError());
  return 0;
}

// zero-bordered fp16 map -> split map (an fp16 value is a TF32 number: lo = 0)
__global__ void k_f16map_to_split(const __half* __restrict__ src, int H, int W, int C, float* __restrict__ dst, int Cd) {
  const int cv = C / 4;
  const long long total = (long long)H * W * cv;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % cv) * 4;
    const long long pix = i / cv;
    const int x = (int)(pix % W), y = (int)(pix / W);
    const uint2 r = *reinterpret_cast<const uint2*>(src + sprow(y, x, W) * C + c);
    const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&r.x)), b = __half22float2(*reinterpret_cast<const __half2*>(&r.y));
    store_split4(dst + sprow(y, x, W) * 2 * Cd, Cd, c, make_float4(a.x, a.y, b.x, b.y));
  }
}
int solo_f16map_to_split(const __half* src, int H, int W, int C, float* dst, int Cdst, cudaStream_t s) {
  k_f16map_to_split<<<device_sm_count() * 4, 256, 0, s>>>(src, H, W, C, dst, Cdst);
  PRISMA_CUDA_OK(cudaGetLastError());
  return 0;
}

// GroupNorm + ReLU apply of a conv output x (dense fp32 [H*W][C], statistics in `stats` as k_gn_final writes them) into
//   out_split : zero-bordered split map (C channels), and / or
//   out_w3    : dense rows [H*W][3 C] = [hi | hi | lo] -- the mask features as the "weight" operand of the dynamic conv
__global__ void k_gn_apply_split(const float* __restrict__ x, int H, int W, int C, const float* __restrict__ stats,
                                 const float* __restrict__ gamma, const float* __restrict__ beta, float* __restrict__ out_split,
                                 float* __restrict__ out_w3) {
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
    const float4 ov = make_float4(o[0], o[1], o[2], o[3]);
    if (out_split) store_split4(out_split + sprow(yy, xx, W) * 2 * C, C, c4, ov);
    if (out_w3) {
      float* row = out_w3 + (size_t)pix * 3 * C;
      const float4 hi = make_float4(tf32_hi(ov.x), tf32_hi(ov.y), tf32_hi(ov.z), tf32_hi(ov.w));
      *reinterpret_cast<float4*>(row + c4) = hi;
      *reinterpret_cast<float4*>(row + C + c4) = hi;
      *reinterpret_cast<float4*>(row + 2 * C + c4) = make_float4(ov.x - hi.x, ov.y - hi.y, ov.z - hi.z, ov.w - hi.w);
    }
  }
}
// declared in solo_kernels.cu (shared statistics kernels)
int gn_stats(const float* x, int HW, int C, int groups, float* part, float* stats, cudaStream_t s);
int groupnorm_relu_split(const float* x, int H, int W, int C, int groups, const float* gamma, const float* beta, float* part,
                         float* stats, float* out_split, float* out_w3, cudaStream_t s) {
  PRISMA_TRY(gn_stats(x, H * W, C, groups, part, stats, s));
  k_gn_apply_split<<<device_sm_count() * 4, 256, 0, s>>>(x, H, W, C, stats, gamma, beta, out_split, out_w3);
  PRISMA_CUDA_OK(cudaGetLastError());
  return 0;
}

// stacked-grid GroupNorm + ReLU (see k_gn_grid): split-map output [B][(F+2)^2][2 C]
__global__ void k_gn_grid_split(const float* __restrict__ x, int F, GridSizes S, int C, int groups, const float* __restrict__ gamma,
                                const float* __restrict__ beta, float* __restrict__ out) {
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
  float* ob = out + (size_t)b * (F + 2) * (F + 2) * 2 * C;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const int c = i % cpg, p = i / cpg, yy = p / Sb, xx = p - yy * Sb;
    const float v = xb[(size_t)(yy * F + xx) * C + c];
    const float o = fmaxf(fmaf((v - mu) * rstd, gamma[g * cpg + c], beta[g * cpg + c]), 0.f);
    float* row = ob + sprow(yy, xx, F) * 2 * C;
    const float hi = tf32_hi(o);
    row[g * cpg + c] = hi;
    row[C + g * cpg + c] = o - hi;
  }
}
int groupnorm_relu_grid_split(const float* x, int B, int F, GridSizes S, int C, int groups, const float* gamma, const float* beta,
                              float* out_split, cudaStream_t s) {
  k_gn_grid_split<<<dim3(groups, B), 256, 0, s>>>(x, F, S, C, groups, gamma, beta, out_split);
  PRISMA_CUDA_OK(cudaGetLastError());
  return 0;
}

// F.interpolate(bilinear, align_corners=False) between split maps (see k_resize_bilinear); Cs source channels are
// interpolated into a map with Cd >= Cs (+2 with coord) channels; coord appends generate_coordinate of the source grid
__device__ __forceinline__ float linspace_m1_1_x(int i, int n) {
  if (n == 1) return -1.f;
  const float step = 2.f / (float)(n - 1);
  return i < n / 2 ? -1.f + step * (float)i : 1.f - step * (float)(n - 1 - i);
}
__global__ void k_resize_bilinear_split(const float* __restrict__ src, int Hs, int Ws, int Cs, int Csp, float* __restrict__ dst, int Hd,
                                        int Wd, int Cd, float sy, float sx, int coord, int accumulate, int Wdf) {
  const int cv = Cs / 4 + (coord ? 1 : 0);
  const long long total = (long long)Hd * Wd * cv;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c4 = (int)(i % cv);
    const int x = (int)((i / cv) % Wd), y = (int)(i / ((long long)cv * Wd));
    const float fy = fmaxf(sy * (y + 0.5f) - 0.5f, 0.f), fx = fmaxf(sx * (x + 0.5f) - 0.5f, 0.f);
    const int y0 = (int)fy, x0 = (int)fx;
    const int y1 = y0 + (y0 < Hs - 1 ? 1 : 0), x1 = x0 + (x0 < Ws - 1 ? 1 : 0);
    const float ly = fy - y0, lx = fx - x0, hy = 1.f - ly, hx = 1.f - lx;
    float* d = dst + sprow(y, x, Wdf) * 2 * Cd;
    if (c4 * 4 >= Cs) {  // the two coordinate channels (+ two zero channels of the 4-vector)
      const float cx = hy * (hx * linspace_m1_1_x(x0, Ws) + lx * linspace_m1_1_x(x1, Ws)) + ly * (hx * linspace_m1_1_x(x0, Ws) + lx * linspace_m1_1_x(x1, Ws));
      const float cy = hy * (hx * linspace_m1_1_x(y0, Hs) + lx * linspace_m1_1_x(y0, Hs)) + ly * (hx * linspace_m1_1_x(y1, Hs) + lx * linspace_m1_1_x(y1, Hs));
      store_split4(d, Cd, Cs, make_float4(cx, cy, 0.f, 0.f));
      continue;
    }
    const int c = c4 * 4;
    const float4 a = load_split4(src + sprow(y0, x0, Ws) * 2 * Csp, Csp, c), b = load_split4(src + sprow(y0, x1, Ws) * 2 * Csp, Csp, c);
    const float4 e = load_split4(src + sprow(y1, x0, Ws) * 2 * Csp, Csp, c), f = load_split4(src + sprow(y1, x1, Ws) * 2 * Csp, Csp, c);
    float4 v;
    v.x = hy * (hx * a.x + lx * b.x) + ly * (hx * e.x + lx * f.x);
    v.y = hy * (hx * a.y + lx * b.y) + ly * (hx * e.y + lx * f.y);
    v.z = hy * (hx * a.z + lx * b.z) + ly * (hx * e.z + lx * f.z);
    v.w = hy * (hx * a.w + lx * b.w) + ly * (hx * e.w + lx * f.w);
    if (accumulate) {
      const float4 p = load_split4(d, Cd, c);
      v.x = p.x + v.x; v.y = p.y + v.y; v.z = p.z + v.z; v.w = p.w + v.w;  // the reference adds the up-sampled map to the sum
    }
    store_split4(d, Cd, c, v);
  }
}
int resize_bilinear_split(const float* src, int Hs, int Ws, int Csrc, int Csrc_pitch, float* dst, int Hd, int Wd, int Cdst, int coord,
                          int accumulate, cudaStream_t s, int dst_frame_w) {
  k_resize_bilinear_split<<<device_sm_count() * 4, 256, 0, s>>>(src, Hs, Ws, Csrc, Csrc_pitch, dst, Hd, Wd, Cdst, (float)Hs / (float)Hd,
                                                 (float)Ws / (float)Wd, coord, accumulate, dst_frame_w > 0 ? dst_frame_w : Wd);
  PRISMA_CUDA_OK(cudaGetLastError());
  return 0;
}

// kernel_preds[inds[:, 0]] as split rows [cap][2 C] (the A operand of the dynamic-conv 3xTF32 GEMM)
__global__ void k_solo_gather_split(const SoloCand* __restrict__ cand, const int* __restrict__ count, int cap,
                                    const float* const* __restrict__ lvl_kernels, const int* __restrict__ lvl_cell0, int levels,
                                    int NC, int C, float* __restrict__ out, const int* __restrict__ lvl_S, int F) {
  const int r = blockIdx.x;
  const int n = min(*count, cap);
  float* o = out + (size_t)r * 2 * C;
  if (r >= n) {
    for (int c = threadIdx.x; c < 2 * C; c += blockDim.x) o[c] = 0.f;
    return;
  }
  const int cell = cand[r].flat / NC;
  int lvl = 0;
  while (lvl + 1 < levels && cell >= lvl_cell0[lvl + 1]) ++lvl;
  int local = cell - lvl_cell0[lvl];
  if (lvl_S) { const int S = lvl_S[lvl]; local = (local / S) * F + local % S; }
  const float* k = lvl_kernels[lvl] + (size_t)local * C;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const float v = k[c], hi = tf32_hi(v);
    o[c] = hi;
    o[C + c] = v - hi;
  }
}
int solo_gather_kernels_split(const SoloCand* cand, const int* count, int cap, const float* const* lvl_kernels,
                              const int* lvl_cell0, int levels, int num_classes, int C, float* out, cudaStream_t s,
                              const int* lvl_S, int frame) {
  k_solo_gather_split<<<cap, 64, 0, s>>>(cand, count, cap, lvl_kernels, lvl_cell0, levels, num_classes, C, out, lvl_S, frame);
  PRISMA_CUDA_OK(cudaGetLastError());
  return 0;
}

// ================================================================ fp32-class backbone (variant "<name>-exact")
// The ResNet + FPN in the same arithmetic as the head: every conv is a 3xTF32 GEMM from a split map to a dense fp32
// [H*W][Cout] output (BatchNorm folded into fp32 weights and bias, ReLU / the residual sum in the epilogue); the kernels
// below are what sits between those GEMMs.  Reference: models/backbones/resnet.py:361-367,631-646, models/necks/fpn.py:151-204.

// stem im2col of the normalised CHW fp32 image for conv1 = Conv2d(3, 64, 7, stride 2, padding 3): row = [hi(192) | lo(192)],
// k = (c*7 + ky)*8 + kx (kx = 7 and k >= 168 zero) -- the K order of raft_im2col_stem, in fp32 halves
__global__ void k_im2col_stem_split(const float* __restrict__ x, int H, int W, float* __restrict__ out) {
  const int Ho = H / 2, Wo = W / 2;
  const long long total = (long long)Ho * Wo * 24;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int g = (int)(i % 24);
    const long long pix = i / 24;
    float v[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (g < 21) {
      const int oy = (int)(pix / Wo), ox = (int)(pix - (long long)oy * Wo);
      const int c = g / 7, ky = g - c * 7;
      const int iy = oy * 2 - 3 + ky, ix0 = ox * 2 - 3;
      if (iy >= 0 && iy < H) {
        const float* row = x + ((size_t)c * H + iy) * W;
#pragma unroll
        for (int j = 0; j < 7; ++j) if (ix0 + j >= 0 && ix0 + j < W) v[j] = __ldg(row + ix0 + j);
      }
    }
    float* o = out + (size_t)pix * 384;
    store_split4(o, 192, g * 8, make_float4(v[0], v[1], v[2], v[3]));
    store_split4(o, 192, g * 8 + 4, make_float4(v[4], v[5], v[6], v[7]));
  }
}
int solo_im2col_stem_split(const float* x, int H, int W, float* out, cudaStream_t s) {
  k_im2col_stem_split<<<device_sm_count() * 8, 256, 0, s>>>(x, H, W, out);
  PRISMA_CUDA_OK(cudaGetLastError());
  return 0;
}

// MaxPool2d(3, stride 2, padding 1) of a dense fp32 NHWC map -> dense fp32 (the identity of the first block) + split map
__global__ void k_maxpool3s2_dense(const float* __restrict__ in, int H, int W, int C, float* __restrict__ out, float* __restrict__ out_split,
                                   int Ho, int Wo) {
  const int cv = C / 4;
  const long long total = (long long)Ho * Wo * cv;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % cv) * 4;
    const int ox = (int)((i / cv) % Wo), oy = (int)(i / ((long long)cv * Wo));
    float4 m = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
    for (int dy = -1; dy <= 1; ++dy)
      for (int dx = -1; dx <= 1; ++dx) {
        const int y = 2 * oy + dy, x = 2 * ox + dx;
        if (y < 0 || y >= H || x < 0 || x >= W) continue;
        const float4 v = *reinterpret_cast<const float4*>(in + ((size_t)y * W + x) * C + c);
        m.x = fmaxf(m.x, v.x); m.y = fmaxf(m.y, v.y); m.z = fmaxf(m.z, v.z); m.w = fmaxf(m.w, v.w);
      }
    *reinterpret_cast<float4*>(out + ((size_t)oy * Wo + ox) * C + c) = m;
    store_split4(out_split + sprow(oy, ox, Wo) * 2 * C, C, c, m);
  }
}
int maxpool3s2_dense(const float* in, int H, int W, int C, float* out, float* out_split, int Ho, int Wo, cudaStream_t s) {
  k_maxpool3s2_dense<<<device_sm_count() * 8, 256, 0, s>>>(in, H, W, C, out, out_split, Ho, Wo);
  PRISMA_CUDA_OK(cudaGetLastError());
  return 0;
}

// FPN top-down step on dense fp32 maps: fine += F.interpolate(coarse, size=fine.shape, mode="nearest") (fpn.py:166-177)
__global__ void k_nearest_add_dense(float* __restrict__ fine, int Hf, int Wf, const float* __restrict__ coarse, int Hc, int Wc, int C,
                                    float sy, float sx) {
  const int cv = C / 4;
  const long long total = (long long)Hf * Wf * cv;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % cv) * 4;
    const int x = (int)((i / cv) % Wf), y = (int)(i / ((long long)cv * Wf));
    const int ys = min((int)floorf(y * sy), Hc - 1), xs = min((int)floorf(x * sx), Wc - 1);
    float4* a = reinterpret_cast<float4*>(fine + ((size_t)y * Wf + x) * C + c);
    const float4 b = *reinterpret_cast<const float4*>(coarse + ((size_t)ys * Wc + xs) * C + c);
    float4 v = *a;
    v.x += b.x; v.y += b.y; v.z += b.z; v.w += b.w;
    *a = v;
  }
}
int nearest_add_dense(float* fine, int Hf, int Wf, const float* coarse, int Hc, int Wc, int C, cudaStream_t s) {
  k_nearest_add_dense<<<device_sm_count() * 4, 256, 0, s>>>(fine, Hf, Wf, coarse, Hc, Wc, C, (float)Hc / (float)Hf, (float)Wc / (float)Wf);
  PRISMA_CUDA_OK(cudaGetLastError());
  return 0;
}

// extra FPN level on dense fp32 maps: F.max_pool2d(x, 1, stride=2) = x[::2, ::2] (fpn.py:188)
__global__ void k_subsample2_dense(const float* __restrict__ in, int W, int C, float* __restrict__ out, int Ho, int Wo) {
  const int cv = C / 4;
  const long long total = (long long)Ho * Wo * cv;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % cv) * 4;
    const int x = (int)((i / cv) % Wo), y = (int)(i / ((long long)cv * Wo));
    *reinterpret_cast<float4*>(out + ((size_t)y * Wo + x) * C + c) = *reinterpret_cast<const float4*>(in + ((size_t)(2 * y) * W + 2 * x) * C + c);
  }
}
int subsample2_dense(const float* in, int H, int W, int C, float* out, int Ho, int Wo, cudaStream_t s) {
  (void)H;
  k_subsample2_dense<<<64, 256, 0, s>>>(in, W, C, out, Ho, Wo);
  PRISMA_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace prisma
