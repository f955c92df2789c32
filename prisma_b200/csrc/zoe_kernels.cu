// prisma_b200 -- pointwise kernels of the ZoeDepth metric head on the Depth-Anything core (bands/depth_anything.py:106-119,
// bands/patchfusion/zoedepth/models/zoedepth/zoedepth_v1.py:127-211).  Everything GEMM-shaped (the 1x1 convs of the
// projectors / regressors / attractor MLPs) runs on the wgmma core; these are the HBM-bound pieces in between.
#include "zoe_kernels.cuh"

#include <math.h>

namespace prisma {

// ---- transforms.ToTensor() (u8 / 255 in f32), core.prep: bilinear(align_corners=True) to 392 x 518, ImageNet normalise
// (base_models/depth_anything.py:171-189).  torch: src = dst * (in-1)/(out-1), f32 lerp weights.
__global__ void k_zoe_preprocess(const uint8_t* __restrict__ img, int H, int W, float* __restrict__ out, int h, int w, float sy,
                                 float sx) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= w) return;
  const float fy = sy * y, fx = sx * x;
  const int y0 = (int)fy, x0 = (int)fx;
  const int y1 = y0 + (y0 < H - 1 ? 1 : 0), x1 = x0 + (x0 < W - 1 ? 1 : 0);
  const float ly = fy - y0, lx = fx - x0, hy = 1.f - ly, hx = 1.f - lx;
  const float mean[3] = {0.485f, 0.456f, 0.406f}, stdv[3] = {0.229f, 0.224f, 0.225f};
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float a = __fdiv_rn((float)img[((size_t)y0 * W + x0) * 3 + c], 255.f), b = __fdiv_rn((float)img[((size_t)y0 * W + x1) * 3 + c], 255.f);
    const float d = __fdiv_rn((float)img[((size_t)y1 * W + x0) * 3 + c], 255.f), e = __fdiv_rn((float)img[((size_t)y1 * W + x1) * 3 + c], 255.f);
    const float v = hy * (hx * a + lx * b) + ly * (hx * d + lx * e);
    out[((size_t)c * h + y) * w + x] = __fdiv_rn(__fsub_rn(v, mean[c]), stdv[c]);
  }
}
int zoe_preprocess(const uint8_t* rgb, int H, int W, float* out_chw, int h, int w, cudaStream_t s) {
  dim3 grid(ceil_div(w, 128), h);
  k_zoe_preprocess<<<grid, 128, 0, s>>>(rgb, H, W, out_chw, h, w, h > 1 ? (float)(H - 1) / (h - 1) : 0.f,
                                        w > 1 ? (float)(W - 1) / (w - 1) : 0.f);
  PRISMA_CUDA_OK(cudaGetLastError());
  return 0;
}

struct AcTap { int i00, i01, i10, i11; float w00, w01, w10, w11; };
__device__ __forceinline__ AcTap ac_tap(int y, int x, int Hs, int Ws, float sy, float sx) {
  const float fy = sy * y, fx = sx * x;
  const int y0 = (int)fy, x0 = (int)fx;
  const int y1 = y0 + (y0 < Hs - 1 ? 1 : 0), x1 = x0 + (x0 < Ws - 1 ? 1 : 0);
  const float ly = fy - y0, lx = fx - x0, hy = 1.f - ly, hx = 1.f - lx;
  AcTap t;
  t.i00 = y0 * Ws + x0; t.i01 = y0 * Ws + x1; t.i10 = y1 * Ws + x0; t.i11 = y1 * Ws + x1;
  t.w00 = hy * hx; t.w01 = hy * lx; t.w10 = ly * hx; t.w11 = ly * lx;
  return t;
}
// torch evaluates h0*(w0*a + w1*b) + h1*(w0*c + w1*d); keep that association
#define AC_EVAL(a, b, c, d, hy, hx, ly, lx) ((hy) * ((hx) * (a) + (lx) * (b)) + (ly) * ((hx) * (c) + (lx) * (d)))

__global__ void k_zoe_embed_add(const float* __restrict__ a, int H, int W, int C, const float* __restrict__ prev, int Hp, int Wp,
                                float sy, float sx, __half* __restrict__ out) {
  const int cv = C / 4;
  const long long total = (long long)H * W * cv;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c4 = (int)(i % cv) * 4;
    const long long pix = i / cv;
    const int x = (int)(pix % W), y = (int)(pix / W);
    const float fy = sy * y, fx = sx * x;
    const int y0 = (int)fy, x0 = (int)fx;
    const int y1 = y0 + (y0 < Hp - 1 ? 1 : 0), x1 = x0 + (x0 < Wp - 1 ? 1 : 0);
    const float ly = fy - y0, lx = fx - x0, hy = 1.f - ly, hx = 1.f - lx;
    const float4 p00 = *reinterpret_cast<const float4*>(prev + ((size_t)y0 * Wp + x0) * C + c4);
    const float4 p01 = *reinterpret_cast<const float4*>(prev + ((size_t)y0 * Wp + x1) * C + c4);
    const float4 p10 = *reinterpret_cast<const float4*>(prev + ((size_t)y1 * Wp + x0) * C + c4);
    const float4 p11 = *reinterpret_cast<const float4*>(prev + ((size_t)y1 * Wp + x1) * C + c4);
    const float4 v = *reinterpret_cast<const float4*>(a + (size_t)pix * C + c4);
    const float o0 = v.x + AC_EVAL(p00.x, p01.x, p10.x, p11.x, hy, hx, ly, lx), o1 = v.y + AC_EVAL(p00.y, p01.y, p10.y, p11.y, hy, hx, ly, lx);
    const float o2 = v.z + AC_EVAL(p00.z, p01.z, p10.z, p11.z, hy, hx, ly, lx), o3 = v.w + AC_EVAL(p00.w, p01.w, p10.w, p11.w, hy, hx, ly, lx);
    *reinterpret_cast<uint2*>(out + (size_t)pix * C + c4) = make_uint2(pack_half2(o0, o1), pack_half2(o2, o3));
  }
}
int zoe_embed_add(const float* a, int H, int W, int C, const float* prev, int Hp, int Wp, __half* out, cudaStream_t s) {
  k_zoe_embed_add<<<device_sm_count() * 4, 256, 0, s>>>(a, H, W, C, prev, Hp, Wp, H > 1 ? (float)(Hp - 1) / (H - 1) : 0.f,
                                         W > 1 ? (float)(Wp - 1) / (W - 1) : 0.f, out);
  PRISMA_CUDA_OK(cudaGetLastError());
  return 0;
}

// attractor.py:165-207 with inv_attractor's defaults alpha = 300, gamma = 2 (the layer never forwards its own alpha), mean
__global__ void k_zoe_attractor(const float* __restrict__ A, int lda, int n_attr, const float* __restrict__ b_prev, int Hp, int Wp,
                                int H, int W, int bins, float sy, float sx, float* __restrict__ b_out) {
  const long long total = (long long)H * W * bins;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int k = (int)(i % bins);
    const long long pix = i / bins;
    const int x = (int)(pix % W), y = (int)(pix / W);
    const float fy = sy * y, fx = sx * x;
    const int y0 = (int)fy, x0 = (int)fx;
    const int y1 = y0 + (y0 < Hp - 1 ? 1 : 0), x1 = x0 + (x0 < Wp - 1 ? 1 : 0);
    const float ly = fy - y0, lx = fx - x0, hy = 1.f - ly, hx = 1.f - lx;
    const float b = AC_EVAL(b_prev[((size_t)y0 * Wp + x0) * bins + k], b_prev[((size_t)y0 * Wp + x1) * bins + k],
                            b_prev[((size_t)y1 * Wp + x0) * bins + k], b_prev[((size_t)y1 * Wp + x1) * bins + k], hy, hx, ly, lx);
    float acc = 0.f;
    for (int a = 0; a < n_attr; ++a) {
      const float dx = A[(size_t)pix * lda + a] - b;
      acc += dx / (1.f + 300.0f * (dx * dx));
    }
    b_out[i] = b + acc / (float)n_attr;
  }
}
int zoe_attractor(const float* A, int lda, int n_attr, const float* b_prev, int Hp, int Wp, int H, int W, int bins, float* b_out,
                  cudaStream_t s) {
  k_zoe_attractor<<<device_sm_count() * 4, 256, 0, s>>>(A, lda, n_attr, b_prev, Hp, Wp, H, W, bins, H > 1 ? (float)(Hp - 1) / (H - 1) : 0.f,
                                         W > 1 ? (float)(Wp - 1) / (W - 1) : 0.f, b_out);
  PRISMA_CUDA_OK(cudaGetLastError());
  return 0;
}

__global__ void k_zoe_concat(const __half* __restrict__ act32, const float* __restrict__ rel, const float* __restrict__ emb, int He,
                             int We, int H, int W, float sy, float sx, __half* __restrict__ out) {
  // one warp per pixel: lanes 0..3 copy the 32 activations (8 each), lane 4 the relative depth, all 32 lanes 4 embedding
  // channels each
  const long long total = (long long)H * W;
  const int lane = threadIdx.x & 31;
  for (long long pix = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; pix < total; pix += ((long long)gridDim.x * blockDim.x) >> 5) {
    const int x = (int)(pix % W), y = (int)(pix / W);
    __half* o = out + (size_t)pix * 192;
    if (lane < 4) *reinterpret_cast<uint4*>(o + lane * 8) = *reinterpret_cast<const uint4*>(act32 + (size_t)pix * 32 + lane * 8);
    if (lane == 4) o[32] = __float2half_rn(rel[pix]);
    const float fy = sy * y, fx = sx * x;
    const int y0 = (int)fy, x0 = (int)fx;
    const int y1 = y0 + (y0 < He - 1 ? 1 : 0), x1 = x0 + (x0 < We - 1 ? 1 : 0);
    const float ly = fy - y0, lx = fx - x0, hy = 1.f - ly, hx = 1.f - lx;
    const int c4 = lane * 4;
    const float4 p00 = *reinterpret_cast<const float4*>(emb + ((size_t)y0 * We + x0) * 128 + c4);
    const float4 p01 = *reinterpret_cast<const float4*>(emb + ((size_t)y0 * We + x1) * 128 + c4);
    const float4 p10 = *reinterpret_cast<const float4*>(emb + ((size_t)y1 * We + x0) * 128 + c4);
    const float4 p11 = *reinterpret_cast<const float4*>(emb + ((size_t)y1 * We + x1) * 128 + c4);
    // channels 33..160 of the 161-channel operand: not 8-byte aligned -> scalar stores
    o[33 + c4 + 0] = __float2half_rn(AC_EVAL(p00.x, p01.x, p10.x, p11.x, hy, hx, ly, lx));
    o[33 + c4 + 1] = __float2half_rn(AC_EVAL(p00.y, p01.y, p10.y, p11.y, hy, hx, ly, lx));
    o[33 + c4 + 2] = __float2half_rn(AC_EVAL(p00.z, p01.z, p10.z, p11.z, hy, hx, ly, lx));
    o[33 + c4 + 3] = __float2half_rn(AC_EVAL(p00.w, p01.w, p10.w, p11.w, hy, hx, ly, lx));
    if (lane < 31) o[161 + lane] = __float2half_rn(0.f);
  }
}
int zoe_concat(const __half* act32, const float* rel, const float* emb, int He, int We, int H, int W, __half* out, cudaStream_t s) {
  k_zoe_concat<<<device_sm_count() * 8, 256, 0, s>>>(act32, rel, emb, He, We, H, W, H > 1 ? (float)(He - 1) / (H - 1) : 0.f,
                                      W > 1 ? (float)(We - 1) / (W - 1) : 0.f, out);
  PRISMA_CUDA_OK(cudaGetLastError());
  return 0;
}

// ConditionalLogBinomial tail + LogBinomial (dist_layers.py:28-63,97-108) + sum(prob * centres) (zoedepth_v1.py:196-199):
// one warp per pixel, two bins per lane.
__global__ void k_zoe_final(const float* __restrict__ pt, const float* __restrict__ centers, int Hc, int Wc, int H, int W, float sy,
                            float sx, float min_temp, float max_temp, float* __restrict__ out) {
  const long long total = (long long)H * W;
  const int lane = threadIdx.x & 31;
  for (long long pix = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; pix < total; pix += ((long long)gridDim.x * blockDim.x) >> 5) {
    const int x = (int)(pix % W), y = (int)(pix / W);
    const float4 q = *reinterpret_cast<const float4*>(pt + (size_t)pix * 4);  // softplus outputs
    const float p0 = q.x + 1e-4f, p1 = q.y + 1e-4f, t0 = q.z + 1e-4f, t1 = q.w + 1e-4f;
    const float p = p0 / (p0 + p1);
    const float t = (max_temp - min_temp) * (t0 / (t0 + t1)) + min_temp;
    const float omx = fminf(fmaxf(1.f - p, 1e-4f), 1.f), px = fminf(fmaxf(p, 1e-4f), 1.f);
    const float lp = logf(px), lq = logf(omx);
    const float fy = sy * y, fx = sx * x;
    const int y0 = (int)fy, x0 = (int)fx;
    const int y1 = y0 + (y0 < Hc - 1 ? 1 : 0), x1 = x0 + (x0 < Wc - 1 ? 1 : 0);
    const float ly = fy - y0, lx = fx - x0, hy = 1.f - ly, hx = 1.f - lx;
    float yv[2], cv[2];
    const float n = 63.f + 1e-7f;
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int k = lane * 2 + j;
      const float kk = (float)k + 1e-7f;
      const float lb = n * logf(n) - kk * logf(kk) - (n - kk) * logf(n - kk + 1e-7f);
      yv[j] = (lb + (float)k * lp + (float)(63 - k) * lq) / t;
      cv[j] = AC_EVAL(centers[((size_t)y0 * Wc + x0) * 64 + k], centers[((size_t)y0 * Wc + x1) * 64 + k],
                      centers[((size_t)y1 * Wc + x0) * 64 + k], centers[((size_t)y1 * Wc + x1) * 64 + k], hy, hx, ly, lx);
    }
    const float mx = warp_max(fmaxf(yv[0], yv[1]));
    const float e0 = expf(yv[0] - mx), e1 = expf(yv[1] - mx);
    const float den = warp_sum(e0 + e1);
    const float num = warp_sum((e0 / den) * cv[0] + (e1 / den) * cv[1]);
    if (lane == 0) out[pix] = num;
  }
}
int zoe_final(const float* pt, const float* centers, int Hc, int Wc, int H, int W, int bins, float min_temp, float max_temp,
              float* out, cudaStream_t s) {
  PRISMA_CHECK(bins == 64, "zoe: 64 bins expected");
  k_zoe_final<<<device_sm_count() * 8, 256, 0, s>>>(pt, centers, Hc, Wc, H, W, H > 1 ? (float)(Hc - 1) / (H - 1) : 0.f,
                                     W > 1 ? (float)(Wc - 1) / (W - 1) : 0.f, min_temp, max_temp, out);
  PRISMA_CUDA_OK(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------------------
// Pillow ImagingResample (src/libImaging/Resample.c) for mode "F", BICUBIC (a = -0.5, support 2): per output index
// center = (i + 0.5) * scale, support = 2 * max(scale, 1), taps [xmin, xmax), weights filter((x + xmin - center + 0.5) /
// filterscale) normalised by their sum, all in double; the horizontal pass runs first and its result is stored as f32.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ double pil_bicubic(double x) {
  const double a = -0.5;
  if (x < 0.0) x = -x;
  if (x < 1.0) return ((a + 2.0) * x - (a + 3.0)) * x * x + 1;
  if (x < 2.0) return (((x - 5) * x + 8) * x - 4) * a;
  return 0.0;
}
__device__ __forceinline__ float pil_resample_1d(const float* __restrict__ src, int stride, int in_size, int out_idx, double scale) {
  const double filterscale = scale < 1.0 ? 1.0 : scale;
  const double support = 2.0 * filterscale;
  const double center = (out_idx + 0.5) * scale;
  const double ss = 1.0 / filterscale;
  int xmin = (int)(center - support + 0.5);
  if (xmin < 0) xmin = 0;
  int xmax = (int)(center + support + 0.5);
  if (xmax > in_size) xmax = in_size;
  xmax -= xmin;
  double ww = 0.0;
  for (int x = 0; x < xmax; ++x) ww += pil_bicubic((x + xmin - center + 0.5) * ss);
  double acc = 0.0;
  for (int x = 0; x < xmax; ++x) {
    double w = pil_bicubic((x + xmin - center + 0.5) * ss);
    if (ww != 0.0) w /= ww;
    acc += (double)src[(size_t)(x + xmin) * stride] * w;
  }
  return (float)acc;
}
__global__ void k_pil_h(const float* __restrict__ in, int ih, int iw, float* __restrict__ tmp, int ow, double scale) {
  const long long total = (long long)ih * ow;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int y = (int)(i / ow), x = (int)(i - (long long)y * ow);
    tmp[i] = pil_resample_1d(in + (size_t)y * iw, 1, iw, x, scale);
  }
}
__global__ void k_pil_v(const float* __restrict__ tmp, int ih, int ow, float* __restrict__ out, int oh, double scale) {
  const long long total = (long long)oh * ow;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int y = (int)(i / ow), x = (int)(i - (long long)y * ow);
    out[i] = pil_resample_1d(tmp + x, ow, ih, y, scale);
  }
}
int pil_bicubic_resize_f32(const float* in, int ih, int iw, float* tmp, float* out, int oh, int ow, cudaStream_t s) {
  k_pil_h<<<device_sm_count() * 8, 256, 0, s>>>(in, ih, iw, tmp, ow, (double)iw / (double)ow);
  k_pil_v<<<device_sm_count() * 8, 256, 0, s>>>(tmp, ih, ow, out, oh, (double)ih / (double)oh);
  PRISMA_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace prisma
