// prisma_b200 -- declarations of the HBM-bound kernels (see pointwise.cu / flow_pointwise.cu).
#pragma once
#include "common.cuh"

namespace prisma {

const char* get_last_error();

// Depth-Anything pre/post (K1, K2a, K3, K4, K8, K10 of SURVEY.md section 2b)
int da_preprocess(const uint8_t* img, int H, int W, float* out_chw, int h, int w, cudaStream_t s, int midas_norm = 0);
int da_patchify(const float* x_chw, int batch, int h, int w, __half* out, int kpad, cudaStream_t s, int patch = 14);
int da_pos_embed(const float* pos, const float* cls, int S, int D, int ph, int pw, float* out, cudaStream_t s);
int layernorm_f16(const float* x, const float* g, const float* b, __half* y, int rows, int D, float eps,
                  cudaStream_t s, int skip_per = 0);
int upsample_ac_f16(const __half* in, int batch, int ih, int iw, int C, __half* out, int oh, int ow, __half* out_relu,
                    cudaStream_t s);
int depth_postprocess(const float* depth, int hn, int wn, int H, int W, int flip, float* pred_out, uint8_t* rgb_out,
                      uint32_t* mm_scratch, float* minmax_out, int num_sms, cudaStream_t s);
int depth_encode_only(const float* pred, int H, int W, int flip, uint8_t* rgb_out, uint32_t* mm_scratch,
                      float* minmax_out, int num_sms, cudaStream_t s);
int depth_encode_png(const float* pred, int H, int W, int flip, uint8_t* rgb_out, uint32_t* mm_scratch,
                     unsigned long long* mag_scratch, float* minmax_out, int num_sms, cudaStream_t s);
// write_pcl's point cloud of an H x W prediction: optional flip, 5x5 median (-> blurred, H*W f32), unprojection packed
// with the u8 RGB frame into H*W 15-byte records (x, y, z f32, red, green, blue u8)
int depth_point_cloud(const float* depth, int H, int W, int flip, const uint8_t* rgb, float* blurred, uint8_t* records,
                      uint32_t* mm_scratch, int num_sms, cudaStream_t s);
int readout_concat_f16(const float* x, int batch, int T, int D, __half* out, cudaStream_t s);
int upsample_bicubic_ac_f32(const float* in, int ih, int iw, float* out, int oh, int ow, int num_sms, cudaStream_t s);
int f32_to_f16(const float* a, __half* b, long long n, cudaStream_t s);

}  // namespace prisma
