// prisma_b200 -- Depth-Anything engine declaration (see engine_da.cu).
#pragma once
#include <functional>
#include <map>
#include <string>
#include <vector>

#include "attention.cuh"
#include "gemm_tc.cuh"
#include "pointwise.cuh"
#include "zoe_kernels.cuh"

namespace prisma {

enum StepGroup { G_PRE = 0, G_LINEAR = 1, G_ATTN = 2, G_LN = 3, G_HEAD = 4, G_RESAMPLE = 5, G_POST = 6 };

struct HostTensor { std::vector<int64_t> shape; std::vector<float> data; };
struct BlockW {
  float *n1w, *n1b, *qkv_b, *proj_b, *g1, *n2w, *n2b, *fc1_b, *fc2_b, *g2;
  __half *qkv_w, *proj_w, *fc1_w, *fc2_w;
};
struct RefineW { __half* out_w; float* out_b; __half* c1_w[2]; float* c1_b[2]; __half* c2_w[2]; float* c2_b[2]; };
struct DaWeights {
  float *cls, *pos, *patch_b, *nw, *nb;
  __half* patch_w;
  std::vector<BlockW> blk;
  __half* proj_w[4]; float* proj_b[4];
  __half *rs0_w, *rs1_w, *rs3_w; float *rs0_b, *rs1_b, *rs3_b;
  __half* rn_w[4];
  RefineW ref[4];
  __half* ro_w[4] = {nullptr, nullptr, nullptr, nullptr};  // MiDaS "project" readout Linear(2D -> D)
  float* ro_b[4] = {nullptr, nullptr, nullptr, nullptr};
  __half *oc1_w, *oc2_w; float *oc1_b, *oc2_b, *oc3_w; float oc3_b;
  // ZoeDepth metric head (zoedepth_v1.py:90-125): 1x1 convs as [N_pad][K_pad] fp16 + fp32 bias
  struct Lin { __half* w = nullptr; float* b = nullptr; int n = 0, k = 0; };
  Lin z_conv2, z_seed0, z_seed2, z_sproj0, z_sproj2, z_proj0[4], z_proj2[4], z_att0[4], z_att2[4], z_clb0, z_clb2;
};
struct DaBuffers {
  uint8_t* img; float* net_in; __half* patches; float* pos; float* x; float* tokens_tap; __half* ln; __half* qkv;
  __half* attn; __half* hid; __half* feat[4]; float* depth; float* pred; uint8_t* rgb; uint32_t* mm; float* minmax;
  unsigned long long* mag;  // Sobel-magnitude maximum of the PNG encode
};
struct Tap { const void* p; int a, b, c; int kind; };  // kind 0: f32 [a][b], 1: padded NHWC f16 (H=a,W=b,C=c), 2: f16 [a][b]
struct Step { int group; const char* name; std::function<int(cudaStream_t)> fn; };
struct PMap;

void da_net_size(int W, int H, int* wn, int* hn);
void midas_net_size(int W, int H, int* wn, int* hn, int side = 384);
enum DepthFamily { FAMILY_DA = 0, FAMILY_MIDAS = 1 };

class DepthEngine {
 public:
  ~DepthEngine();
  int init(const std::string& encoder, int device);
  int load_tensor(const std::string& name, const float* data, const int64_t* shape, int ndim);
  int finalize();
  int infer(const uint8_t* rgb, int n, int H, int W, float* depth_out, uint8_t* rgb_out, float* min_out, float* max_out);
  int infer_resident(int H, int W, int n, int iters, float* ms_per_iter);
  int encode(const float* pred, int H, int W, int flip, uint8_t* rgb_out, float* min_out, float* max_out, int png_variant = 0);
  int infer_image(const uint8_t* rgb, int H, int W, float* depth_out, uint8_t* png_rgb_out, float* min_out, float* max_out);
  int point_cloud(const float* pred, int H, int W, int flip, const uint8_t* rgb, uint8_t* records_out);
  int set_net_side(int side);
  long long read_tap(const std::string& name, float* out, long long capacity);
  int profile(int H, int W, int n, float* out8);
  int build_plan(int H, int W, int batch);
  // n frames in passes of `pass_frames`: H2D of pass i+1 and D2H of pass i-1 overlap the compute of pass i
  int infer_stream(const uint8_t* rgb, int n, int H, int W, int pass_frames, float* depth_out, uint8_t* rgb_out,
                   float* min_out, float* max_out);

  bool debug_taps = true;
  double work_linear = 0, work_attn = 0, work_head = 0;
  std::vector<Step> steps;
  int device = 0;

 private:
  const HostTensor* get(const std::string& name, std::initializer_list<int64_t> shape);
  int up_f32(const std::string& name, std::initializer_list<int64_t> shape, float** out, float scale = 1.f, int n_scaled = 0);
  int up_linear(const std::string& name, int N, int K, __half** out, float scale = 1.f, int n_scaled = 0);
  int up_conv(const std::string& name, int Cout, int Cin, int kh, int kw, __half** out);
  int up_convT(const std::string& name, int Cin, int Cout, int s, __half** out, float** bias_out);
  int up_lin1x1(const std::string& name, int N, int K, DaWeights::Lin* out);
  int build_metric_head(const PMap& btlnck, const PMap* r_maps, const __half* act32, int Bt);
  int new_map(PMap* m, int H, int W, int C);
  void add(int group, const char* name, std::function<int(cudaStream_t)> fn);
  int add_gemm(int group, const char* name, const __half* A, long long a_rows, int a_cols, int a_pitch, const __half* W,
               int M, int N, int taps, const int* tap_off, const GemmEpilogue& ep, double flops);
  int add_conv3x3(const char* name, const PMap& in, const __half* W, int Cout, GemmEpilogue ep, int sub,
                  const PMap* out_geom);
  int run_steps(cudaStream_t s);
  int run_steps_direct(cudaStream_t s);

  std::string encoder;
  int D = 0, depth = 0, heads = 0, F = 0, oc[4] = {0, 0, 0, 0};
  // family switches: Depth-Anything (DINOv2 ViT/14 + DPT head) or MiDaS DPT (timm ViT/16, "project" readout, hooks)
  int family = FAMILY_DA, patch = 14, pos_grid = 37, hooks[4] = {0, 0, 0, 0};
  int net_side = 384;  // MiDaS transform side: 384 (hub default_transform) or 256 (small_transform)
  float* zoe_metric = nullptr; float* zoe_tmp = nullptr; int plan_W_req = 0;
  bool metric = false;  // --metric indoor|outdoor: ZoeDepth head on the relative model, fixed 392 x 518 network input
  std::vector<float> host_pos, host_cls;  // MiDaS: pos-embed resized on the host per resolution (bilinear)
  __half* ro_cat = nullptr;               // MiDaS: [B*P][2D] readout operand
  int num_sms = 132;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  // streamed (double-buffered) clip path
  struct StreamSlot {
    uint8_t* in = nullptr; uint8_t* rgb = nullptr; float* pred = nullptr; float* mm = nullptr;
    cudaEvent_t loaded = nullptr, consumed = nullptr, done = nullptr, drained = nullptr;
  } slot[2];
  cudaStream_t s_in = nullptr, s_out = nullptr;
  float* mm_host = nullptr;  // pinned, 2 floats per frame
  size_t mm_host_frames = 0;
  int ensure_stream_slots(int H, int W, int Bt, bool want_pred);
  size_t slot_frames = 0, slot_bytes_frame = 0;
  bool slot_has_pred = false;
  cudaGraphExec_t graph_exec = nullptr;
  bool finalized = false;
  std::map<std::string, HostTensor> host;
  std::vector<void*> allocs, plan_allocs;
  DaWeights w;
  DaBuffers b;
  std::map<std::string, Tap> taps;
  int plan_H = 0, plan_W = 0, batch = 0, hn = 0, wn = 0, ph = 0, pw = 0, T = 0;
};

}  // namespace prisma
