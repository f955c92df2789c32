// prisma_b200 -- SOLOv2 engine declaration (see engine_solo.cu).
#pragma once
#include <functional>
#include <map>
#include <string>
#include <vector>

#include "engine_da.cuh"
#include "solo_kernels.cuh"

namespace prisma {

struct SoloConvW { __half* w = nullptr; float* b = nullptr; float* gn_w = nullptr; float* gn_b = nullptr; int cout = 0, cin = 0, k = 1; };
struct SoloConvW3 { float* w = nullptr; float* b = nullptr; float* gn_w = nullptr; float* gn_b = nullptr; int cout = 0, cin = 0, cin32 = 0, k = 1; };
struct XMap { float* p = nullptr; int H = 0, W = 0, C = 0;   // split map: zero-bordered NHWC rows of 2 C floats [hi | lo] (solo_exact.cu)
              int Hp() const { return H + 2; } int Wp() const { return W + 2; } long long rows() const { return (long long)Hp() * Wp(); } };
struct SMap { __half* p = nullptr; int H = 0, W = 0, C = 0;
              int Hp() const { return H + 2; } int Wp() const { return W + 2; } long long rows() const { return (long long)Hp() * Wp(); } };
struct SoloTap { const void* p; int kind; int a, b, c; };  // kind 0: f32 [a][b], 1: padded f16 map (H=a,W=b,C=c), 2: f16 [a][b], 3: u8 [a][b]

class SoloEngine {
 public:
  ~SoloEngine();
  int init(const std::string& variant, int device);
  int load_tensor(const std::string& name, const float* data, const int64_t* shape, int ndim);
  int finalize();
  // one frame: union mask (H x W u8, the band's frame), kept instances (<= 100): scores, labels, optional masks [n][H][W]
  int infer(const uint8_t* rgb, int H, int W, float confidence, uint8_t* union_out, int* n_out, float* scores_out,
            int* labels_out, uint8_t* inst_masks_out, float* ms_out);
  // Tests: replace FPN level `level` of the NEXT head replay by these values (dense fp32 NCHW [256][h][w]) ...
  int inject_feat(int level, const float* nchw, int h, int w);
  // ... and run head + decode from the injected levels (frame geometry H x W as planned by a previous infer call)
  // img_h / img_w > 0 override the resized-image size used by the final mask crop (meta img_shape, solov2_head.py:751-757)
  int infer_from_feats(int H, int W, int img_h, int img_w, float confidence, uint8_t* union_out, int* n_out, float* scores_out,
                       int* labels_out, uint8_t* inst_masks_out);
  bool exact_head = true;   // fp32-class head + decode (3xTF32 contractions, fp32 activations): the default of the band
  bool exact_backbone = false;  // "<variant>-exact": ResNet + FPN in the same fp32-class arithmetic (3 tensor-core passes per conv)
  long long read_tap(const std::string& name, float* out, long long capacity);
  int net_shape(int H, int W, int* nh, int* nw, int* hp, int* wp) const;
  double flops = 0;
  int launches = 0;
  int device = 0;

 private:
  const HostTensor* get(const std::string& name);
  int up_conv(const std::string& name, const std::string& bn, const std::string& gn, int Cout, int Cin, int k, bool bias,
              SoloConvW* out);
  int build_plan(int H, int W);
  int run(cudaStream_t s);

  std::string variant;
  int layers[4] = {3, 4, 23, 3}, scale_long = 1333, scale_short = 800;
  int num_grids[5] = {40, 36, 24, 16, 12};
  float strides[5] = {8, 8, 16, 32, 32};
  int num_sms = 132;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  cudaGraphExec_t graph_exec = nullptr;
  bool use_graph = true, finalized = false;
  std::map<std::string, HostTensor> host;
  std::vector<void*> allocs, plan_allocs;
  std::vector<std::function<int(cudaStream_t)>> steps;
  std::vector<const char*> step_tag;  // stage of each step (PRISMA_SOLO_PROFILE)
  std::map<std::string, SoloTap> taps;
  // weights
  SoloConvW stem;
  struct Block { SoloConvW c1, c2, c3, ds; bool has_ds = false; int stride = 1; };
  std::vector<Block> blocks[4];
  SoloConvW lateral[4], fpnc[4], mf[4][3], mf_pred, kconv[4], cconv[4], conv_cls, conv_kernel;
  SoloConvW3 mf3[4][3], mf_pred3, kconv3[4], cconv3[4], conv_cls3, conv_kernel3;  // the head in [hi | hi | lo] fp32 (exact_head)
  int up_conv3(const std::string& name, const std::string& gn, int Cout, int Cin, int k, bool bias, SoloConvW3* out,
               const std::string& bn = "");
  SoloConvW3 stem3, lateral3[4], fpnc3[4];  // exact_backbone
  struct Block3 { SoloConvW3 c1, c2, c3, ds; };
  std::vector<Block3> blocks3[4];
  float* d_feat_in[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};  // injected FPN levels, dense fp32 NHWC
  int feat_h[5] = {0, 0, 0, 0, 0}, feat_w[5] = {0, 0, 0, 0, 0};
  bool inject = false;
  size_t head_step0 = 0;           // first step of the head (after the FPN)
  const float* d_masks_f = nullptr;  // exact head: fp32 sigmoid mask predictions [cap][fh*fw]
  // plan state
  int plan_H = 0, plan_W = 0, nh = 0, nw = 0, hp = 0, wp = 0, fh = 0, fw = 0;
  uint8_t* d_img = nullptr; uint8_t* d_resized = nullptr; float* d_net = nullptr;
  uint8_t* d_union = nullptr; uint8_t* d_inst = nullptr;
  float* d_conf = nullptr;
  int *d_count = nullptr, *d_ntop = nullptr, *d_nkeep = nullptr, *d_top = nullptr, *d_keep = nullptr, *d_keep_label = nullptr;
  float* d_keep_score = nullptr;
  const __half* d_masks = nullptr;  // sigmoid mask predictions of the candidates [cap][fh*fw]
};

}  // namespace prisma
