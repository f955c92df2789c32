// prisma_b200 -- RAFT optical-flow engine declaration (see engine_raft.cu).
#pragma once
#include <functional>
#include <map>
#include <string>
#include <vector>

#include "engine_da.cuh"  // HostTensor, Step, Tap
#include "flow.cuh"
#include "raft_kernels.cuh"

namespace prisma {

struct ConvW { __half* w = nullptr; float* b = nullptr; int cout = 0, cin = 0, kh = 1, kw = 1;
               int wsplit = 1; };  // wsplit 2: every tap's K slab is stored twice, [fp16(w) | fp16(w - fp16(w))], the tap is walked twice
struct ResW { ConvW c1, c2, ds; bool has_ds = false; };
struct EncW { ConvW stem; ResW blk[3][2]; ConvW out; };
struct RaftWeights {
  EncW fnet, cnet;
  ConvW convc1, convc2, convf2, conv, zr[2], q[2], fh1, fh2, mk1, mk2;
  float *convf1_w = nullptr, *convf1_b = nullptr;
  ConvW fh2u; float fh2_b[2] = {0.f, 0.f};  // FlowHead.conv2 as a 1x1 conv to 18 per-tap partial products (hi/lo weights)
  __half* convf1_gemm_w = nullptr;  // [256][256]: k = [98 weights | 0 | the same 98 (for the fp16 'lo' half of the flow) | 0]
};
struct RaftBuffers {
  uint8_t* img; uint8_t* resized; float* chw; __half* stem_cols; float *coords0, *coords1, *cnet_out, *h_master, *delta, *mask;
  float* flow_up; uint8_t* rgb; uint32_t* mm; float* maxd; float* h_tap = nullptr; float* coords_tap = nullptr;
};
struct RMap;

class RaftEngine {
 public:
  ~RaftEngine();
  int init(int device);
  int load_tensor(const std::string& name, const float* data, const int64_t* shape, int ndim);
  int finalize();
  // prev/curr: h*w*3 u8 RGB; fwd/bwd: hs*ws*2 f32 (may be NULL); *_rgb: hs*ws*3 u8 (may be NULL)
  // reuse_prev: `prev` is the `curr` of the previous call (a video loop): its fnet / cnet features are reused, only `curr`
  // is uploaded and encoded.  Ignored (full pass) when no valid cache exists.
  int infer(const uint8_t* prev, const uint8_t* curr, int H, int W, double scale, int iters, float* fwd, float* bwd,
            uint8_t* fwd_rgb, uint8_t* bwd_rgb, float* max_fwd, float* max_bwd, float* ms_out, int reuse_prev = 0);
  // The video loop over a chunk of n frames (flow_raft.py:97-115): pair j = (frame j, frame j+1), or with continue_clip
  // (the engine still holds the features of the frame before frames[0]) pair j = (frame j-1, frame j).  Three streams:
  // the upload of frame j+1 and the download of pair j-1 overlap the graph of pair j.  Outputs are pair-major, each may
  // be NULL.  *pairs_out = number of pairs produced.
  int infer_stream(const uint8_t* frames, int n, int H, int W, double scale, int iters, int continue_clip, float* fwd,
                   float* bwd, uint8_t* fwd_rgb, uint8_t* bwd_rgb, float* max_fwd, float* max_bwd, int* pairs_out);
  // `reps` video passes over the frames already on the device (kernel-only leg of bench.py): ms per pass, CUDA events
  int time_resident(int H, int W, double scale, int iters, int reps, float* ms_per_pass);
  long long read_tap(const std::string& name, float* out, long long capacity);
  int build_plan(int H, int W, double scale, int iters);
  int Hs = 0, Ws = 0, H8 = 0, W8 = 0;
  double flops = 0, flops_conv = 0, flops_conv_video = 0;  // full pass total; conv GEMMs of the full / video pass
  int profile(int H, int W, double scale, int iters, float* out8);
  bool has_cache() const { return cache_valid; }
  // Frame pairs per pass of the clip path (infer_stream / time_resident / profile / work_detail): 1..4, default 4
  // (PRISMA_RAFT_PAIRS overrides), see build_plan; clip_pairs() lowers it for frames whose pyramids would not fit.  The pair call infer() always plans one pair per pass; switching
  // between the two paths rebuilds the plan.
  int set_pairs_per_pass(int np);
  int pairs_per_pass() const { return stream_pairs; }
  int use_pairs(int np);  // select the plan variant for the next build_plan
  int clip_pairs(int H, int W, double scale) const;
  int plan_pairs() const { return plan_B / 2; }  // pairs per pass of the current plan
  FlowCorr* corr_block() { return corr; }
  std::vector<Step> steps;
  bool debug_taps = true;

 private:
  const HostTensor* get(const std::string& name);
  int up_conv(const std::string& name, const std::string& bn, int Cout, int Cin, int kh, int kw, int Npad, float out_scale,
              ConvW* out, int wsplit = 1, const std::vector<int>* chans = nullptr, bool with_bias = true);
  int up_encoder(const std::string& prefix, bool bn, EncW* e);
  int new_map(RMap* m, int B, int H, int W, int C, int pad);
  void add(const char* name, std::function<int(cudaStream_t)> fn);
  int add_conv(const char* name, const RMap& in, int c0, const ConvW& cw, GemmEpilogue ep, int sub);
  int add_conv_in(const char* name, const RMap& in, const ConvW& cw, int sub, float* dense, float* stats);
  int build_encoder(const EncW& e, bool inorm, const __half* stem_cols, RMap* out_map128, int B);
  int run_direct(cudaStream_t s, int which = 1);  // which: 1 = full pass, 2 = video pass reusing the previous frame's features

  int device = 0, num_sms = 132;
  cudaStream_t stream = nullptr;
  cudaGraphExec_t graph_exec = nullptr, graph_cached = nullptr;
  int cur_mask = 3;          // steps carry a mask (Step::group): bit 0 = full pass, bit 1 = video pass
  bool cache_valid = false;  // slot NP of the feature buffers holds the last frame of the previous pass
  bool use_graph = true, finalized = false;
  std::map<std::string, HostTensor> host;
  std::vector<void*> allocs, plan_allocs;
  RaftWeights w;
  RaftBuffers b;
  FlowCorr* corr = nullptr;
  std::map<std::string, Tap> taps;
  float *dense_a = nullptr, *dense_b = nullptr, *stats_a = nullptr, *stats_b = nullptr, *in_part = nullptr;
  float* slab_part = nullptr; double* slab_part2 = nullptr; size_t slab_part_floats = 0;
  int npairs = 1, stream_pairs = 4, plan_B = 2;
  size_t device_mem = 0;
  int plan_H = 0, plan_W = 0, iters = 0, Hp_ = 0, Wp_ = 0, pads[4] = {0, 0, 0, 0};
  double plan_scale = 0.0;
  struct StreamSlot {
    uint8_t* in = nullptr; float* flow = nullptr; uint8_t* rgb = nullptr; float* mx = nullptr;
    cudaEvent_t loaded = nullptr, consumed = nullptr, done = nullptr, drained = nullptr;
  } slot[2];
  cudaStream_t s_in = nullptr, s_out = nullptr;
  float* mx_host = nullptr;  // pinned, 2 floats per pair (padded to whole passes)
  size_t mx_host_pairs = 0, slot_in_bytes = 0, slot_out_px = 0;
  int ensure_stream_slots(int H, int W);
};

}  // namespace prisma
