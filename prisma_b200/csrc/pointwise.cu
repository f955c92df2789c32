// prisma_b200 -- HBM-bound kernels of the Depth-Anything path: pre-process (OpenCV-exact cubic resize + normalise),
// patchify, pos-embed interpolation, LayerNorm, bilinear resamplers, min/max + heat encode.
// All of these are memory/latency bound: coalesced 16-byte accesses, one pass where possible, warp-shuffle reductions.
#include "pointwise.cuh"

namespace prisma {

// ------------------------------------------------------------------------------------------------
// K1: u8 RGB HxWx3  ->  f32 CHW net input, bit-faithful to
//   image = img/255.0 (f64); cv2.resize(image,(w,h),INTER_CUBIC); (image-mean)/std (f64); astype(f32)
// (bands/depth_anything.py:122-126, d_anything/util/transform.py:168-174,219-222,232-234).
// OpenCV's cubic for CV_64F: tap weights in *float* (A=-0.75, 4th = 1 - sum), source coordinate
// fx = (float)((dx+0.5)*scale - 0.5), horizontal then vertical pass in double, replicate border, no FMA.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void cv_cubic_coeffs(float x, float* c) {
  const float A = -0.75f;
  c[0] = __fsub_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fsub_rn(__fmul_rn(A, __fadd_rn(x, 1.f)), __fmul_rn(5.f, A)), __fadd_rn(x, 1.f)), __fmul_rn(8.f, A)), __fadd_rn(x, 1.f)), __fmul_rn(4.f, A));
  c[1] = __fadd_rn(__fmul_rn(__fmul_rn(__fsub_rn(__fmul_rn(__fadd_rn(A, 2.f), x), __fadd_rn(A, 3.f)), x), x), 1.f);
  const float y = __fsub_rn(1.f, x);
  c[2] = __fadd_rn(__fmul_rn(__fmul_rn(__fsub_rn(__fmul_rn(__fadd_rn(A, 2.f), y), __fadd_rn(A, 3.f)), y), y), 1.f);
  c[3] = __fsub_rn(__fsub_rn(__fsub_rn(1.f, c[0]), c[1]), c[2]);
}

struct MeanStd { double mean[3], stdv[3]; };

__global__ void k_da_preprocess(const uint8_t* __restrict__ img, int H, int W, float* __restrict__ out, int h, int w,
                                double scale_x, double scale_y, MeanStd ms) {
  const int ox = blockIdx.x * blockDim.x + threadIdx.x;
  const int oy = blockIdx.y;
  if (ox >= w) return;
  float fx = (float)__dsub_rn(__dmul_rn((double)ox + 0.5, scale_x), 0.5);
  int sx = (int)floorf(fx);
  fx = __fsub_rn(fx, (float)sx);
  float fy = (float)__dsub_rn(__dmul_rn((double)oy + 0.5, scale_y), 0.5);
  int sy = (int)floorf(fy);
  fy = __fsub_rn(fy, (float)sy);
  float cx[4], cy[4];
  cv_cubic_coeffs(fx, cx);
  cv_cubic_coeffs(fy, cy);
  int xs[4], ys[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    xs[k] = min(max(sx - 1 + k, 0), W - 1);
    ys[k] = min(max(sy - 1 + k, 0), H - 1);
  }
  double acc[3] = {0.0, 0.0, 0.0};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const uint8_t* row = img + (size_t)ys[j] * W * 3;
    double hsum[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      // D[dx] = S[-1]*a0 + S[0]*a1 + S[1]*a2 + S[2]*a3, left to right, double x float->double
      double s = __dmul_rn(__ddiv_rn((double)row[xs[0] * 3 + c], 255.0), (double)cx[0]);
      s = __dadd_rn(s, __dmul_rn(__ddiv_rn((double)row[xs[1] * 3 + c], 255.0), (double)cx[1]));
      s = __dadd_rn(s, __dmul_rn(__ddiv_rn((double)row[xs[2] * 3 + c], 255.0), (double)cx[2]));
      s = __dadd_rn(s, __dmul_rn(__ddiv_rn((double)row[xs[3] * 3 + c], 255.0), (double)cx[3]));
      hsum[c] = s;
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const double t = __dmul_rn(hsum[c], (double)cy[j]);
      acc[c] = (j == 0) ? t : __dadd_rn(acc[c], t);
    }
  }
#pragma unroll
  for (int c = 0; c < 3; ++c)
    out[((size_t)c * h + oy) * w + ox] = (float)__ddiv_rn(__dsub_rn(acc[c], ms.mean[c]), ms.stdv[c]);
}

int da_preprocess(const uint8_t* img, int H, int W, float* out, int h, int w, cudaStream_t s, int midas_norm) {
  dim3 block(128), grid(ceil_div(w, 128), h);
  // cv::resize: inv_scale = dsize/ssize ; scale = 1./inv_scale
  const double scale_x = 1.0 / ((double)w / (double)W);
  const double scale_y = 1.0 / ((double)h / (double)H);
  // NormalizeImage: ImageNet statistics, for Depth-Anything (depth_anything.py:72) and for the hubconf default_transform the
  // MiDaS band selects (depth_midas.py:37-40); midas_norm == 2 would be upstream's dpt_transform (mean = std = 0.5), unused
  const MeanStd ms = midas_norm == 2 ? MeanStd{{0.5, 0.5, 0.5}, {0.5, 0.5, 0.5}} : MeanStd{{0.485, 0.456, 0.406}, {0.229, 0.224, 0.225}};
  k_da_preprocess<<<grid, block, 0, s>>>(img, H, W, out, h, w, scale_x, scale_y, ms);
  PRISMA_CUDA_OK(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------------------
// K2a: patchify  f32 CHW [3][h][w] -> fp16 [P][kpad]  (k = c*196 + ky*14 + kx, zero padded to kpad)
// = im2col of the 14x14/stride-14 patch-embed conv (dinov2/layers/patch_embed.py:66,76-78).
// ------------------------------------------------------------------------------------------------
__global__ void k_patchify(const float* __restrict__ x_all, int h, int w, __half* __restrict__ out, int pw, int kpad,
                           int per_img, int ps) {
  const int img = blockIdx.x / per_img;
  const int p = blockIdx.x;             // output row (image-major)
  const int pl = p - img * per_img;     // patch index inside the image
  const float* x = x_all + (size_t)img * 3 * h * w;
  const int py = pl / pw, px = pl - py * pw;
  for (int k = threadIdx.x; k < kpad; k += blockDim.x) {
    float v = 0.f;
    if (k < 3 * ps * ps) {
      const int c = k / (ps * ps), r = k - c * ps * ps, ky = r / ps, kx = r - ky * ps;
      v = x[((size_t)c * h + py * ps + ky) * w + px * ps + kx];
    }
    out[(size_t)p * kpad + k] = __float2half_rn(v);
  }
}
int da_patchify(const float* x, int batch, int h, int w, __half* out, int kpad, cudaStream_t s, int patch) {
  const int ph = h / patch, pw = w / patch;
  k_patchify<<<batch * ph * pw, 160, 0, s>>>(x, h, w, out, pw, kpad, ph * pw, patch);
  PRISMA_CUDA_OK(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------------------
// K3: pos-embed interpolation (once per resolution): F.interpolate(bicubic, scale_factor=((ph+.1)/S,(pw+.1)/S))
// of the SxS grid (vision_transformer.py:179-210).  torch semantics: src = (dst+0.5)*(1/scale_factor) - 0.5 in
// float, A=-0.75, the four taps evaluated independently, clamped reads.  out[0] = pos[0] + cls.
// Square-grid rule: when the grid is already S x S (ph == pw == S), interpolate_pos_encoding returns the table unchanged
// (vision_transformer.py:183-184) -- a resample with scale factor (S+0.1)/S would not be the identity -- so da_pos_embed
// copies rows 1..S*S bit for bit and launches only the block of row 0.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float cubic1(float x, float A) { return ((A + 2.f) * x - (A + 3.f)) * x * x + 1.f; }
__device__ __forceinline__ float cubic2(float x, float A) { return ((A * x - 5.f * A) * x + 8.f * A) * x - 4.f * A; }

__global__ void k_pos_embed(const float* __restrict__ pos, const float* __restrict__ cls, int S, int D, int ph, int pw,
                            float rscale_y, float rscale_x, float* __restrict__ out) {
  const int t = blockIdx.x;  // token
  if (t == 0) {
    for (int d = threadIdx.x; d < D; d += blockDim.x) out[d] = pos[d] + cls[d];
    return;
  }
  const int oy = (t - 1) / pw, ox = (t - 1) - oy * pw;
  const float A = -0.75f;
  const float ry = rscale_y * (oy + 0.5f) - 0.5f;
  const float rx = rscale_x * (ox + 0.5f) - 0.5f;
  const int iy = (int)floorf(ry), ix = (int)floorf(rx);
  const float ty = ry - iy, tx = rx - ix;
  float wy[4] = {cubic2(ty + 1.f, A), cubic1(ty, A), cubic1(1.f - ty, A), cubic2(2.f - ty, A)};
  float wx[4] = {cubic2(tx + 1.f, A), cubic1(tx, A), cubic1(1.f - tx, A), cubic2(2.f - tx, A)};
  for (int d = threadIdx.x; d < D; d += blockDim.x) {
    float acc = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int yy = min(max(iy - 1 + j, 0), S - 1);
      float r = 0.f;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int xx = min(max(ix - 1 + i, 0), S - 1);
        r += pos[(size_t)(1 + yy * S + xx) * D + d] * wx[i];
      }
      acc += r * wy[j];
    }
    out[(size_t)t * D + d] = acc;
  }
}
int da_pos_embed(const float* pos, const float* cls, int S, int D, int ph, int pw, float* out, cudaStream_t s) {
  // torch: scale = (float)(1.0 / scale_factor), scale_factor = (p + 0.1) / S computed in double
  const float rsy = (float)(1.0 / ((double)(ph + 0.1) / (double)S));
  const float rsx = (float)(1.0 / ((double)(pw + 0.1) / (double)S));
  const bool square = ph == S && pw == S;
  k_pos_embed<<<square ? 1 : 1 + ph * pw, 128, 0, s>>>(pos, cls, S, D, ph, pw, rsy, rsx, out);
  PRISMA_CUDA_OK(cudaGetLastError());
  if (square) PRISMA_CUDA_OK(cudaMemcpyAsync(out + D, pos + D, (size_t)S * S * D * sizeof(float), cudaMemcpyDeviceToDevice, s));
  return 0;
}

// ------------------------------------------------------------------------------------------------
// K4: LayerNorm fp32 [rows][D] -> fp16 [rows][D]; one warp per row, row held in registers (D <= 1024).
// ------------------------------------------------------------------------------------------------
template <int V4>  // float4 per lane: D = 128 * V4
__global__ void k_layernorm(const float* __restrict__ x, const float* __restrict__ g, const float* __restrict__ b,
                            __half* __restrict__ y, int rows, float eps, int skip_per) {
  constexpr int D = 128 * V4;
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  // skip_per > 0: output row r = b*skip_per + p reads input row b*(skip_per+1) + 1 + p (drops each image's cls token)
  const int src = skip_per > 0 ? row + row / skip_per + 1 : row;
  const float4* xr = reinterpret_cast<const float4*>(x + (size_t)src * D);
  float4 v[V4];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < V4; ++i) {
    v[i] = xr[lane + 32 * i];
    s += v[i].x + v[i].y + v[i].z + v[i].w;
  }
  const float mean = warp_sum(s) * (1.0f / D);
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < V4; ++i) {
    const float a = v[i].x - mean, bb = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
    q += a * a + bb * bb + c * c + d * d;
  }
  const float rstd = rsqrtf(warp_sum(q) * (1.0f / D) + eps);
  uint2* yr = reinterpret_cast<uint2*>(y + (size_t)row * D);
#pragma unroll
  for (int i = 0; i < V4; ++i) {
    const float4 gg = reinterpret_cast<const float4*>(g)[lane + 32 * i];
    const float4 bb = reinterpret_cast<const float4*>(b)[lane + 32 * i];
    uint2 o;
    o.x = pack_half2((v[i].x - mean) * rstd * gg.x + bb.x, (v[i].y - mean) * rstd * gg.y + bb.y);
    o.y = pack_half2((v[i].z - mean) * rstd * gg.z + bb.z, (v[i].w - mean) * rstd * gg.w + bb.w);
    yr[lane + 32 * i] = o;
  }
}
int layernorm_f16(const float* x, const float* g, const float* b, __half* y, int rows, int D, float eps,
                  cudaStream_t s, int skip_per) {
  const int wpb = 8;
  dim3 grid(ceil_div(rows, wpb)), block(32 * wpb);
  switch (D) {
    case 384: k_layernorm<3><<<grid, block, 0, s>>>(x, g, b, y, rows, eps, skip_per); break;
    case 768: k_layernorm<6><<<grid, block, 0, s>>>(x, g, b, y, rows, eps, skip_per); break;
    case 1024: k_layernorm<8><<<grid, block, 0, s>>>(x, g, b, y, rows, eps, skip_per); break;
    default: set_last_error("layernorm: unsupported D"); return -1;
  }
  PRISMA_CUDA_OK(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------------------
// K8: bilinear resize, align_corners=True, zero-bordered NHWC fp16 -> zero-bordered NHWC fp16
// (F.interpolate in FeatureFusionBlock, d_anything/blocks.py:141-147 and dpt.py:133).
// torch: scale=(in-1)/(out-1) (float), src=scale*dst, i0=(int)src, i1=i0+(i0<in-1), l1=src-i0, l0=1-l1.
// 8 channels (16 B) per thread.
// ------------------------------------------------------------------------------------------------
__global__ void k_upsample_ac(const __half* __restrict__ in_all, int ih, int iw, int C, __half* __restrict__ out_all,
                              int oh, int ow, float sy, float sx, int relu_copy, __half* __restrict__ out_relu_all) {
  // grid = (ceil(ow * C/8 / 256), oh, batch): the row and the image come from the block index, so the only division per
  // thread is a 32-bit one by C/8
  const __half* in = in_all + (size_t)blockIdx.z * (ih + 2) * (iw + 2) * C;
  __half* out = out_all + (size_t)blockIdx.z * (oh + 2) * (ow + 2) * C;
  __half* out_relu = relu_copy ? out_relu_all + (size_t)blockIdx.z * (oh + 2) * (ow + 2) * C : nullptr;
  const unsigned c8 = (unsigned)C >> 3;
  const unsigned t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (unsigned)ow * c8) return;
  const int ox = (int)(t / c8), c = (int)(t - (unsigned)ox * c8);
  const int oy = blockIdx.y;
  const float fy = sy * oy, fx = sx * ox;
  const int y0 = (int)fy, x0 = (int)fx;
  const int y1 = y0 + (y0 < ih - 1 ? 1 : 0), x1 = x0 + (x0 < iw - 1 ? 1 : 0);
  const float ly1 = fy - y0, ly0 = 1.f - ly1, lx1 = fx - x0, lx0 = 1.f - lx1;
  const int iwp = iw + 2, owp = ow + 2;
  const __half* r0 = in + ((size_t)(y0 + 1) * iwp + 1) * C + c * 8;
  const __half* r1 = in + ((size_t)(y1 + 1) * iwp + 1) * C + c * 8;
  const uint4 a = *reinterpret_cast<const uint4*>(r0 + (size_t)x0 * C), b = *reinterpret_cast<const uint4*>(r0 + (size_t)x1 * C);
  const uint4 cc = *reinterpret_cast<const uint4*>(r1 + (size_t)x0 * C), d = *reinterpret_cast<const uint4*>(r1 + (size_t)x1 * C);
  const __half2* ha = reinterpret_cast<const __half2*>(&a);
  const __half2* hb = reinterpret_cast<const __half2*>(&b);
  const __half2* hc = reinterpret_cast<const __half2*>(&cc);
  const __half2* hd = reinterpret_cast<const __half2*>(&d);
  uint32_t o[4], orl[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 fa = __half22float2(ha[j]), fb = __half22float2(hb[j]), fc = __half22float2(hc[j]),
                 fd = __half22float2(hd[j]);
    const float r0v = ly0 * (lx0 * fa.x + lx1 * fb.x) + ly1 * (lx0 * fc.x + lx1 * fd.x);
    const float r1v = ly0 * (lx0 * fa.y + lx1 * fb.y) + ly1 * (lx0 * fc.y + lx1 * fd.y);
    o[j] = pack_half2(r0v, r1v);
    orl[j] = pack_half2(fmaxf(r0v, 0.f), fmaxf(r1v, 0.f));
  }
  const size_t off = ((size_t)(oy + 1) * owp + ox + 1) * C + c * 8;
  *reinterpret_cast<uint4*>(out + off) = make_uint4(o[0], o[1], o[2], o[3]);
  if (relu_copy) *reinterpret_cast<uint4*>(out_relu + off) = make_uint4(orl[0], orl[1], orl[2], orl[3]);
}
int upsample_ac_f16(const __half* in, int batch, int ih, int iw, int C, __half* out, int oh, int ow, __half* out_relu,
                    cudaStream_t s) {
  PRISMA_CHECK(C % 8 == 0, "upsample: C must be a multiple of 8");
  const float sy = oh > 1 ? (float)(ih - 1) / (float)(oh - 1) : 0.f;
  const float sx = ow > 1 ? (float)(iw - 1) / (float)(ow - 1) : 0.f;
  const unsigned per_row = (unsigned)ow * (unsigned)(C / 8);
  k_upsample_ac<<<dim3((per_row + 255) / 256, oh, batch), 256, 0, s>>>(
      in, ih, iw, C, out, oh, ow, sy, sx, out_relu != nullptr, out_relu);
  PRISMA_CUDA_OK(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------------------
// K10: depth post-process (bands/depth_anything.py:132,215-220; common/encode.py:13-33)
//   pass 1: prediction = bilinear(align_corners=False) of the hn x wn net depth to H x W ; global min / max
//   pass 2: d = (p-min)/(max-min) [f32]; d = 1-d [f32]; rgb = trunc(255 * hue_to_rgb((1-d)*0.65)) in f64
// The source (1.9 MB) stays in L2 between the passes; the passes write H*W*4 (optional) and H*W*3 bytes.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float bilinear_af(const float* __restrict__ d, int hn, int wn, float sy, float sx, int oy,
                                             int ox) {
  // torch area_pixel_compute_source_index(align_corners=False): max(scale*(dst+0.5)-0.5, 0)
  const float fy = fmaxf(sy * (oy + 0.5f) - 0.5f, 0.f), fx = fmaxf(sx * (ox + 0.5f) - 0.5f, 0.f);
  const int y0 = (int)fy, x0 = (int)fx;
  const int y1 = y0 + (y0 < hn - 1 ? 1 : 0), x1 = x0 + (x0 < wn - 1 ? 1 : 0);
  const float ly1 = fy - y0, ly0 = 1.f - ly1, lx1 = fx - x0, lx0 = 1.f - lx1;
  return ly0 * (lx0 * d[(size_t)y0 * wn + x0] + lx1 * d[(size_t)y0 * wn + x1]) +
         ly1 * (lx0 * d[(size_t)y1 * wn + x0] + lx1 * d[(size_t)y1 * wn + x1]);
}
// order-preserving float <-> uint mapping so atomicMin/Max work on floats of either sign
__device__ __forceinline__ uint32_t f2ord(float f) {
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float ord2f(uint32_t u) {
  return __uint_as_float((u & 0x80000000u) ? (u & 0x7FFFFFFFu) : ~u);
}

__global__ void k_minmax_init(uint32_t* mm) { mm[0] = 0xFFFFFFFFu; mm[1] = 0u; }

__global__ void k_depth_upsample_minmax(const float* __restrict__ d, int hn, int wn, float* __restrict__ pred, int H,
                                        int W, float sy, float sx, uint32_t* __restrict__ mm) {
  float lo = INFINITY, hi = -INFINITY;
  const long long total = (long long)H * W;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int oy = (int)(i / W), ox = (int)(i - (long long)oy * W);
    const float v = bilinear_af(d, hn, wn, sy, sx, oy, ox);
    if (pred) pred[i] = v;
    lo = fminf(lo, v);
    hi = fmaxf(hi, v);
  }
  lo = warp_min(lo);
  hi = warp_max(hi);
  __shared__ float slo[32], shi[32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) { slo[warp] = lo; shi[warp] = hi; }
  __syncthreads();
  if (warp == 0) {
    const int nw = blockDim.x >> 5;
    lo = lane < nw ? slo[lane] : INFINITY;
    hi = lane < nw ? shi[lane] : -INFINITY;
    lo = warp_min(lo);
    hi = warp_max(hi);
    if (lane == 0) { atomicMin(&mm[0], f2ord(lo)); atomicMax(&mm[1], f2ord(hi)); }
  }
}

__device__ __forceinline__ uint8_t hue_channel_u8(double hue6, double off) {
  // trunc(255 * clip(|mod(6*hue + off, 6) - 3| - 1, 0, 1)), every op rounded separately (numpy f64 semantics)
  double v = fmod(__dadd_rn(hue6, off), 6.0);
  v = __dsub_rn(fabs(__dsub_rn(v, 3.0)), 1.0);
  v = fmin(fmax(v, 0.0), 1.0);
  return (uint8_t)(int)__dmul_rn(v, 255.0);
}

__global__ void k_depth_encode(const float* __restrict__ d, int hn, int wn, const float* __restrict__ pred_in, int H,
                               int W, float sy, float sx, const uint32_t* __restrict__ mm, int flip,
                               uint8_t* __restrict__ rgb, float* __restrict__ minmax_out) {
  const float dmin = ord2f(mm[0]), dmax = ord2f(mm[1]);
  if (blockIdx.x == 0 && threadIdx.x == 0 && minmax_out) { minmax_out[0] = dmin; minmax_out[1] = dmax; }
  const float range = __fsub_rn(dmax, dmin);
  const long long total = (long long)H * W;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    float p;
    if (pred_in) p = pred_in[i];
    else { const int oy = (int)(i / W), ox = (int)(i - (long long)oy * W); p = bilinear_af(d, hn, wn, sy, sx, oy, ox); }
    float x = __fdiv_rn(__fsub_rn(p, dmin), range);
    if (flip & 1) x = __fsub_rn(1.0f, x);
    // heat_to_rgb(h) = hue_to_rgb((1-h)*0.65); rgb = hue*6 + {0,4,2}
    uint8_t* o = rgb + i * 3;
    if (flip & 2) {
      // depth_midas.py:144 passes the f32 array: (1-h)*0.65, *6 and +{4,2} round in f32 before the f64 rgb array
      const float hue6 = __fmul_rn(__fmul_rn(__fsub_rn(1.0f, x), 0.65f), 6.0f);
      o[0] = hue_channel_u8((double)hue6, 0.0);
      o[1] = hue_channel_u8((double)__fadd_rn(hue6, 4.0f), 0.0);
      o[2] = hue_channel_u8((double)__fadd_rn(hue6, 2.0f), 0.0);
    } else {  // depth_anything.py:219 casts to f64 first
      const double hue = __dmul_rn(__dsub_rn(1.0, (double)x), 0.65);
      const double hue6 = __dmul_rn(hue, 6.0);
      o[0] = hue_channel_u8(hue6, 0.0);
      o[1] = hue_channel_u8(hue6, 4.0);
      o[2] = hue_channel_u8(hue6, 2.0);
    }
  }
}

int depth_postprocess(const float* depth, int hn, int wn, int H, int W, int flip, float* pred_out, uint8_t* rgb_out,
                      uint32_t* mm_scratch, float* minmax_out, int num_sms, cudaStream_t s) {
  // torch area_pixel_compute_scale(align_corners=False): (float)in / out
  const float sy = (float)hn / (float)H, sx = (float)wn / (float)W;
  k_minmax_init<<<1, 1, 0, s>>>(mm_scratch);
  const int grid = num_sms * 8;
  k_depth_upsample_minmax<<<grid, 256, 0, s>>>(depth, hn, wn, pred_out, H, W, sy, sx, mm_scratch);
  k_depth_encode<<<grid, 256, 0, s>>>(depth, hn, wn, pred_out, H, W, sy, sx, mm_scratch, flip, rgb_out, minmax_out);
  PRISMA_CUDA_OK(cudaGetLastError());
  return 0;
}

// encode only, from a given H x W prediction (used by the parity tests to pin the encoder bit-exactly)
__global__ void k_minmax_plain(const float* __restrict__ p, long long n, uint32_t* __restrict__ mm) {
  float lo = INFINITY, hi = -INFINITY;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    lo = fminf(lo, p[i]);
    hi = fmaxf(hi, p[i]);
  }
  lo = warp_min(lo);
  hi = warp_max(hi);
  if ((threadIdx.x & 31) == 0) { atomicMin(&mm[0], f2ord(lo)); atomicMax(&mm[1], f2ord(hi)); }
}
int depth_encode_only(const float* pred, int H, int W, int flip, uint8_t* rgb_out, uint32_t* mm_scratch,
                      float* minmax_out, int num_sms, cudaStream_t s) {
  k_minmax_init<<<1, 1, 0, s>>>(mm_scratch);
  k_minmax_plain<<<num_sms * 4, 256, 0, s>>>(pred, (long long)H * W, mm_scratch);
  k_depth_encode<<<num_sms * 8, 256, 0, s>>>(nullptr, 0, 0, pred, H, W, 0.f, 0.f, mm_scratch, flip, rgb_out, minmax_out);
  PRISMA_CUDA_OK(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------------------
// PNG variant of the depth encode = write_depth(normalize, heatmap, encode_range) (bands/common/io.py:138-166), used by
// process_image (bands/depth_anything.py:173): heat map whose saturation carries the Sobel edges of the u8 depth image
// (common/encode.py:81-95, ksize=1 -> [-1,0,1], BORDER_REFLECT_101) and whose pixels (0,0),(0,1) carry (min,max) packed
// in 24 bits over [0,1000] (encode.py:141-146, evaluated in f32 exactly as numpy does).
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ int depth_u8(const float* __restrict__ p, int W, int y, int x, float dmin, float range, int flip) {
  float d = __fdiv_rn(__fsub_rn(p[(size_t)y * W + x], dmin), range);
  if (flip) d = __fsub_rn(1.0f, d);
  return (int)(uint8_t)(int)__fmul_rn(d, 255.0f);
}
__device__ __forceinline__ double sobel_mag(const float* __restrict__ p, int H, int W, int y, int x, float dmin, float range,
                                            int flip) {
  const int xl = x > 0 ? x - 1 : (W > 1 ? 1 : 0), xr = x < W - 1 ? x + 1 : (W > 1 ? W - 2 : 0);
  const int yu = y > 0 ? y - 1 : (H > 1 ? 1 : 0), yd = y < H - 1 ? y + 1 : (H > 1 ? H - 2 : 0);
  const double sx = (double)(depth_u8(p, W, y, xr, dmin, range, flip) - depth_u8(p, W, y, xl, dmin, range, flip));
  const double sy = (double)(depth_u8(p, W, yd, x, dmin, range, flip) - depth_u8(p, W, yu, x, dmin, range, flip));
  return sqrt(__dadd_rn(__dmul_rn(sx, sx), __dmul_rn(sy, sy)));
}
__global__ void k_sobel_max(const float* __restrict__ p, int H, int W, const uint32_t* __restrict__ mm, int flip,
                            unsigned long long* __restrict__ magmax) {
  const float dmin = ord2f(mm[0]), range = __fsub_rn(ord2f(mm[1]), dmin);
  double hi = 0.0;
  const long long total = (long long)H * W;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int y = (int)(i / W), x = (int)(i - (long long)y * W);
    hi = fmax(hi, sobel_mag(p, H, W, y, x, dmin, range, flip));
  }
  for (int o = 16; o > 0; o >>= 1) hi = fmax(hi, __shfl_xor_sync(0xffffffffu, hi, o));
  if ((threadIdx.x & 31) == 0) atomicMax(magmax, (unsigned long long)__double_as_longlong(hi));  // hi >= 0
}
__device__ __forceinline__ void range_pixel(float value, uint8_t* o) {
  // float_to_rgb(value, 0, 1000): numpy keeps everything in f32 (256^3 - 1 = 2^24 - 1 is exactly representable)
  const float L = __fmul_rn(fminf(fmaxf(__fdiv_rn(value, 1000.0f), 0.0f), 1.0f), 16777215.0f);
  const float c0 = __fdiv_rn(floorf(fmodf(L, 256.0f)), 255.0f);
  const float c1 = __fdiv_rn(fmodf(floorf(__fdiv_rn(L, 256.0f)), 256.0f), 255.0f);
  const float c2 = __fdiv_rn(fmodf(floorf(__fdiv_rn(L, 65536.0f)), 256.0f), 255.0f);
  o[0] = (uint8_t)(int)__dmul_rn((double)c0, 255.0);
  o[1] = (uint8_t)(int)__dmul_rn((double)c1, 255.0);
  o[2] = (uint8_t)(int)__dmul_rn((double)c2, 255.0);
}
__device__ __forceinline__ uint8_t heat_sat_u8(double hue6, double off, double sat, double one_minus_sat) {
  double v = fmod(__dadd_rn(hue6, off), 6.0);
  v = __dsub_rn(fabs(__dsub_rn(v, 3.0)), 1.0);
  v = fmin(fmax(v, 0.0), 1.0);
  v = __dadd_rn(__dmul_rn(v, sat), one_minus_sat);
  return (uint8_t)(int)__dmul_rn(v, 255.0);
}
__global__ void k_depth_encode_png(const float* __restrict__ p, int H, int W, const uint32_t* __restrict__ mm, int flip,
                                   const unsigned long long* __restrict__ magmax, uint8_t* __restrict__ rgb,
                                   float* __restrict__ minmax_out) {
  const float dmin = ord2f(mm[0]), dmax = ord2f(mm[1]);
  if (blockIdx.x == 0 && threadIdx.x == 0 && minmax_out) { minmax_out[0] = dmin; minmax_out[1] = dmax; }
  const float range = __fsub_rn(dmax, dmin);
  const double k = __ddiv_rn(255.0, __longlong_as_double((long long)*magmax));  // sobel_mag *= 255.0 / sobel_mag.max()
  const long long total = (long long)H * W;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    uint8_t* o = rgb + i * 3;
    if (i == 0) { range_pixel(dmin, o); continue; }
    if (i == 1) { range_pixel(dmax, o); continue; }
    const int y = (int)(i / W), x = (int)(i - (long long)y * W);
    float d = __fdiv_rn(__fsub_rn(p[i], dmin), range);
    if (flip) d = __fsub_rn(1.0f, d);
    const double edge = __ddiv_rn(__dmul_rn(sobel_mag(p, H, W, y, x, dmin, range, flip), k), 255.0);
    const double sat = __dsub_rn(1.0, edge), oms = __dsub_rn(1.0, sat);
    const double hue6 = __dmul_rn(__dmul_rn(__dsub_rn(1.0, (double)d), 0.65), 6.0);
    o[0] = heat_sat_u8(hue6, 0.0, sat, oms);
    o[1] = heat_sat_u8(hue6, 4.0, sat, oms);
    o[2] = heat_sat_u8(hue6, 2.0, sat, oms);
  }
}
__global__ void k_zero_u64(unsigned long long* p) { *p = 0ull; }

int depth_encode_png(const float* pred, int H, int W, int flip, uint8_t* rgb_out, uint32_t* mm_scratch,
                     unsigned long long* mag_scratch, float* minmax_out, int num_sms, cudaStream_t s) {
  k_minmax_init<<<1, 1, 0, s>>>(mm_scratch);
  k_zero_u64<<<1, 1, 0, s>>>(mag_scratch);
  k_minmax_plain<<<num_sms * 4, 256, 0, s>>>(pred, (long long)H * W, mm_scratch);
  k_sobel_max<<<num_sms * 8, 256, 0, s>>>(pred, H, W, mm_scratch, flip, mag_scratch);
  k_depth_encode_png<<<num_sms * 8, 256, 0, s>>>(pred, H, W, mm_scratch, flip, mag_scratch, rgb_out, minmax_out);
  PRISMA_CUDA_OK(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------------------
// Point cloud of a still image = write_pcl (bands/common/io.py:201-211) -> create_point_cloud (common/geom.py:5-24):
//   (a) flip (only when asked): t = (d-min)/(max-min); t = 1-t; d = min + t*(max-min), all f32
//   (b) cv2.medianBlur(d, 5): the 13th of the 25 values of the 5x5 window, BORDER_REPLICATE
//   (c) X = d*((x-W/2)/1000), Y = d*(-((y-H/2)/1000)), Z = d*(-1), f32 -> 15-byte records x y z f4, red green blue u1
// Every f32 operation is rounded separately (__f*_rn), as numpy does, so no FMA contraction can change a bit.
// Per pixel: the median reads 4 B (+ the halo, from shared memory) and writes 4 B; the pack reads 4 + 3 B and writes 15 B.
// ------------------------------------------------------------------------------------------------
constexpr int PCL_TILE = 32, PCL_THREADS_Y = 8, PCL_HALO = 2;
constexpr int PCL_SPAN = PCL_TILE + 2 * PCL_HALO;

__device__ __forceinline__ float pcl_flip(float d, float dmin, float range) {
  const float t = __fsub_rn(1.0f, __fdiv_rn(__fsub_rn(d, dmin), range));
  return __fadd_rn(dmin, __fmul_rn(t, range));
}

// Median of 25: Batcher's odd-even merge sort for 32 inputs, with the comparators that touch inputs 25..31 dropped (padding
// with +inf never moves) and only those that feed position 12 kept: 113 compare-exchanges.  The median of a 5x5 window is a
// value of the window whatever the ties, so any correct selection network gives the reference's bits.
__device__ __forceinline__ float median25(float* v) {
#define CE(i, j) { const float a = v[i], b = v[j]; v[i] = fminf(a, b); v[j] = fmaxf(a, b); }
  CE(0,1) CE(2,3) CE(4,5) CE(6,7) CE(8,9) CE(10,11) CE(12,13) CE(14,15) CE(16,17) CE(18,19) CE(20,21) CE(22,23)
  CE(0,2) CE(1,3) CE(4,6) CE(5,7) CE(8,10) CE(9,11) CE(12,14) CE(13,15) CE(16,18) CE(17,19) CE(20,22) CE(21,23)
  CE(1,2) CE(5,6) CE(9,10) CE(13,14) CE(17,18) CE(21,22) CE(0,4) CE(1,5) CE(2,6) CE(3,7) CE(8,12) CE(9,13) CE(10,14)
  CE(11,15) CE(16,20) CE(17,21) CE(18,22) CE(19,23) CE(2,4) CE(3,5) CE(10,12) CE(11,13) CE(18,20) CE(19,21) CE(1,2)
  CE(3,4) CE(5,6) CE(9,10) CE(11,12) CE(13,14) CE(17,18) CE(19,20) CE(21,22) CE(0,8) CE(1,9) CE(2,10) CE(3,11)
  CE(4,12) CE(5,13) CE(6,14) CE(7,15) CE(16,24) CE(4,8) CE(5,9) CE(6,10) CE(7,11) CE(20,24) CE(2,4) CE(3,5) CE(6,8)
  CE(7,9) CE(10,12) CE(11,13) CE(18,20) CE(19,21) CE(22,24) CE(1,2) CE(3,4) CE(5,6) CE(7,8) CE(9,10) CE(11,12)
  CE(13,14) CE(17,18) CE(19,20) CE(21,22) CE(23,24) CE(0,16) CE(1,17) CE(2,18) CE(3,19) CE(4,20) CE(5,21) CE(6,22)
  CE(7,23) CE(8,24) CE(8,16) CE(9,17) CE(10,18) CE(11,19) CE(12,20) CE(13,21) CE(6,10) CE(7,11) CE(12,16) CE(13,17)
  CE(10,12) CE(11,13) CE(11,12)
#undef CE
  return v[12];
}

// One 32 x 32 output tile per block of 32 x 8 threads: the 36 x 36 input window (replicated borders, flipped on load) is
// staged once in shared memory; each thread selects four medians in registers.
__global__ void __launch_bounds__(PCL_TILE * PCL_THREADS_Y) k_pcl_median5(const float* __restrict__ d, int H, int W,
                                                                          const uint32_t* __restrict__ mm, int flip,
                                                                          float* __restrict__ out) {
  __shared__ float t[PCL_SPAN][PCL_SPAN];
  const int x0 = blockIdx.x * PCL_TILE, y0 = blockIdx.y * PCL_TILE;
  float dmin = 0.f, range = 0.f;
  if (flip) { dmin = ord2f(mm[0]); range = __fsub_rn(ord2f(mm[1]), dmin); }
  const int tid = threadIdx.y * PCL_TILE + threadIdx.x;
  for (int i = tid; i < PCL_SPAN * PCL_SPAN; i += PCL_TILE * PCL_THREADS_Y) {
    const int r = i / PCL_SPAN, c = i - r * PCL_SPAN;
    const int gy = min(max(y0 + r - PCL_HALO, 0), H - 1), gx = min(max(x0 + c - PCL_HALO, 0), W - 1);
    const float v = d[(size_t)gy * W + gx];
    t[r][c] = flip ? pcl_flip(v, dmin, range) : v;
  }
  __syncthreads();
  const int x = x0 + threadIdx.x;
#pragma unroll
  for (int k = 0; k < PCL_TILE / PCL_THREADS_Y; ++k) {
    const int ry = threadIdx.y + k * PCL_THREADS_Y, y = y0 + ry;
    float v[25];
#pragma unroll
    for (int dy = 0; dy < 5; ++dy)
#pragma unroll
      for (int dx = 0; dx < 5; ++dx) v[dy * 5 + dx] = t[ry + dy][threadIdx.x + dx];
    const float m = median25(v);
    if (x < W && y < H) out[(size_t)y * W + x] = m;
  }
}

// 256 pixels per block: the block's 768 colour bytes are staged in shared memory, each thread assembles its 15-byte record
// there, and the block writes its 3840 contiguous record bytes as 16-byte stores (3840 = 240 * 16, so every full block
// starts 16-byte aligned).
constexpr int PCL_PACK = 256;
__global__ void __launch_bounds__(PCL_PACK) k_pcl_unproject_pack(const float* __restrict__ d, const uint8_t* __restrict__ rgb,
                                                                 int H, int W, uint8_t* __restrict__ out) {
  __shared__ __align__(16) uint8_t col[PCL_PACK * 3];
  __shared__ __align__(16) uint8_t rec[PCL_PACK * 15];
  const long long n = (long long)H * W, p0 = (long long)blockIdx.x * PCL_PACK;
  const int cnt = (int)min((long long)PCL_PACK, n - p0);
  const uint8_t* src = rgb + p0 * 3;
  uint8_t* dst = out + p0 * 15;
  if (cnt == PCL_PACK) {
    for (int i = threadIdx.x; i < PCL_PACK * 3 / 16; i += PCL_PACK)
      reinterpret_cast<uint4*>(col)[i] = reinterpret_cast<const uint4*>(src)[i];
  } else {
    for (int i = threadIdx.x; i < cnt * 3; i += PCL_PACK) col[i] = src[i];
  }
  __syncthreads();
  if (threadIdx.x < cnt) {
    const long long p = p0 + threadIdx.x;
    const int y = (int)(p / W), x = (int)(p - (long long)y * W);
    const float dv = d[p];
    const float u0 = 0.5f * (float)W, v0 = 0.5f * (float)H;  // rgb.shape[1] / 2, rgb.shape[0] / 2: exact in f32
    const float xyz[3] = {__fmul_rn(dv, __fdiv_rn(__fsub_rn((float)x, u0), 1000.0f)),
                          __fmul_rn(dv, -__fdiv_rn(__fsub_rn((float)y, v0), 1000.0f)),
                          __fmul_rn(dv, -1.0f)};
    uint8_t* o = rec + threadIdx.x * 15;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const uint32_t b = __float_as_uint(xyz[c]);
#pragma unroll
      for (int k = 0; k < 4; ++k) o[c * 4 + k] = (uint8_t)(b >> (8 * k));
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) o[12 + c] = col[threadIdx.x * 3 + c];
  }
  __syncthreads();
  if (cnt == PCL_PACK) {
    for (int i = threadIdx.x; i < PCL_PACK * 15 / 16; i += PCL_PACK)
      reinterpret_cast<uint4*>(dst)[i] = reinterpret_cast<const uint4*>(rec)[i];
  } else {
    for (int i = threadIdx.x; i < cnt * 15; i += PCL_PACK) dst[i] = rec[i];
  }
}

int depth_point_cloud(const float* depth, int H, int W, int flip, const uint8_t* rgb, float* blurred, uint8_t* records,
                      uint32_t* mm_scratch, int num_sms, cudaStream_t s) {
  PRISMA_CHECK(H > 0 && W > 0, "point cloud: empty frame");
  PRISMA_CHECK(H <= 65535 * PCL_TILE, "point cloud: frame too tall");
  const long long n = (long long)H * W;
  if (flip) {
    k_minmax_init<<<1, 1, 0, s>>>(mm_scratch);
    k_minmax_plain<<<num_sms * 4, 256, 0, s>>>(depth, n, mm_scratch);
  }
  k_pcl_median5<<<dim3((W + PCL_TILE - 1) / PCL_TILE, (H + PCL_TILE - 1) / PCL_TILE), dim3(PCL_TILE, PCL_THREADS_Y), 0, s>>>(
      depth, H, W, mm_scratch, flip, blurred);
  k_pcl_unproject_pack<<<(unsigned)((n + PCL_PACK - 1) / PCL_PACK), PCL_PACK, 0, s>>>(blurred, rgb, H, W, records);
  PRISMA_CUDA_OK(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------------------
// small utilities
// ------------------------------------------------------------------------------------------------
__global__ void k_f32_to_f16(const float* __restrict__ a, __half* __restrict__ b, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) b[i] = __float2half_rn(a[i]);
}
int f32_to_f16(const float* a, __half* b, long long n, cudaStream_t s) {
  k_f32_to_f16<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(a, b, n);
  PRISMA_CUDA_OK(cudaGetLastError());
  return 0;
}


// ------------------------------------------------------------------------------------------------
// MiDaS DPT "project" readout (midas/backbones/utils.py ProjectReadout): A[b*P + p] = [ x[b][1+p] | x[b][0] ] as fp16,
// the operand of Linear(2D -> D) + GELU.
// ------------------------------------------------------------------------------------------------
__global__ void k_readout_concat(const float* __restrict__ x, int T, int D, __half* __restrict__ out) {
  const int P = T - 1;
  const int row = blockIdx.x, b = row / P, p = row - b * P;
  const float* tok = x + ((size_t)b * T + 1 + p) * D;
  const float* cls = x + (size_t)b * T * D;
  __half* o = out + (size_t)row * 2 * D;
  for (int d = threadIdx.x * 4; d < D; d += blockDim.x * 4) {
    const float4 a = *reinterpret_cast<const float4*>(tok + d);
    const float4 c = *reinterpret_cast<const float4*>(cls + d);
    *reinterpret_cast<uint2*>(o + d) = make_uint2(pack_half2(a.x, a.y), pack_half2(a.z, a.w));
    *reinterpret_cast<uint2*>(o + D + d) = make_uint2(pack_half2(c.x, c.y), pack_half2(c.z, c.w));
  }
}
int readout_concat_f16(const float* x, int batch, int T, int D, __half* out, cudaStream_t s) {
  k_readout_concat<<<batch * (T - 1), 128, 0, s>>>(x, T, D, out);
  PRISMA_CUDA_OK(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------------------
// F.interpolate(mode="bicubic", align_corners=True) of one f32 map (bands/depth_midas.py:58-63): torch's
// upsample_bicubic2d: src = dst * (in-1)/(out-1), A = -0.75, clamped taps, fp32 accumulation, rows then columns.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float cubic_interp1d_t(float x0, float x1, float x2, float x3, float t) {
  const float A = -0.75f;
  return x0 * cubic2(t + 1.f, A) + x1 * cubic1(t, A) + x2 * cubic1(1.f - t, A) + x3 * cubic2(2.f - t, A);
}
__global__ void k_upsample_bicubic_ac(const float* __restrict__ in, int ih, int iw, float* __restrict__ out, int oh, int ow,
                                      float sy, float sx) {
  const long long total = (long long)oh * ow;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int oy = (int)(i / ow), ox = (int)(i - (long long)oy * ow);
    const float ry = sy * oy, rx = sx * ox;
    const int iy = (int)floorf(ry), ix = (int)floorf(rx);
    const float ty = ry - iy, tx = rx - ix;
    float r[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float* row = in + (size_t)min(max(iy - 1 + k, 0), ih - 1) * iw;
      r[k] = cubic_interp1d_t(row[min(max(ix - 1, 0), iw - 1)], row[min(max(ix, 0), iw - 1)], row[min(max(ix + 1, 0), iw - 1)],
                              row[min(max(ix + 2, 0), iw - 1)], tx);
    }
    out[i] = cubic_interp1d_t(r[0], r[1], r[2], r[3], ty);
  }
}
int upsample_bicubic_ac_f32(const float* in, int ih, int iw, float* out, int oh, int ow, int num_sms, cudaStream_t s) {
  const float sy = oh > 1 ? (float)(ih - 1) / (float)(oh - 1) : 0.f;
  const float sx = ow > 1 ? (float)(iw - 1) / (float)(ow - 1) : 0.f;
  k_upsample_bicubic_ac<<<num_sms * 8, 256, 0, s>>>(in, ih, iw, out, oh, ow, sy, sx);
  PRISMA_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace prisma
