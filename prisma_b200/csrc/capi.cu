// prisma_b200 -- the C ABI (include/prisma_b200.h).  Nothing throws across it.
#include "../../include/prisma_b200.h"

#include <cstring>
#include <new>
#include <vector>

#include "engine_da.cuh"
#include "engine_raft.cuh"
#include "engine_solo.cuh"
#include "flow.cuh"

using namespace prisma;

struct prisma_engine {
  int kind;  // 1 = depth, 2 = flow correlation, 3 = RAFT
  DepthEngine* depth;
  FlowCorr* corr;
  RaftEngine* raft = nullptr;
  SoloEngine* solo = nullptr;  // kind 4
};

#define API_GUARD_BEGIN try {
#define API_GUARD_END                                                   \
  }                                                                     \
  catch (const std::exception& ex) {                                    \
    set_last_error(std::string("exception: ") + ex.what());             \
    return -3;                                                          \
  }                                                                     \
  catch (...) {                                                         \
    set_last_error("unknown exception");                                \
    return -3;                                                          \
  }

// ------------------------------------------------------------------------------------------------ debug / kernel-level
namespace {
struct Scratch {
  std::vector<void*> p;
  ~Scratch() { for (void* q : p) cudaFree(q); }
  template <typename T>
  T* alloc(size_t n) {
    void* q = nullptr;
    if (cudaMalloc(&q, std::max<size_t>(n * sizeof(T), 256)) != cudaSuccess) return nullptr;
    cudaMemset(q, 0, std::max<size_t>(n * sizeof(T), 256));
    p.push_back(q);
    return reinterpret_cast<T*>(q);
  }
};
int device_sms(int device, int* sms) {
  PRISMA_CUDA_OK(cudaSetDevice(device));
  cudaDeviceProp prop;
  PRISMA_CUDA_OK(cudaGetDeviceProperties(&prop, device));
  PRISMA_CHECK(prop.major == 9 && prop.minor == 0, "prisma_b200 kernels are sm_90a only; there is no fallback path");
  *sms = prop.multiProcessorCount;
  return 0;
}
std::vector<__half> to_half_padded(const float* src, int rows, int cols, int rows_pad, int cols_pad) {
  std::vector<__half> h((size_t)rows_pad * cols_pad, __float2half_rn(0.f));
  for (int r = 0; r < rows; ++r)
    for (int c = 0; c < cols; ++c) h[(size_t)r * cols_pad + c] = __float2half_rn(src[(size_t)r * cols + c]);
  return h;
}
int timed(cudaStream_t s, int iters, float* ms_out, const std::function<int()>& fn) {
  cudaEvent_t a, b;
  PRISMA_CUDA_OK(cudaEventCreate(&a));
  PRISMA_CUDA_OK(cudaEventCreate(&b));
  PRISMA_TRY(fn());  // warm
  PRISMA_CUDA_OK(cudaEventRecord(a, s));
  for (int i = 0; i < iters; ++i) PRISMA_TRY(fn());
  PRISMA_CUDA_OK(cudaEventRecord(b, s));
  PRISMA_CUDA_OK(cudaStreamSynchronize(s));
  float ms = 0;
  PRISMA_CUDA_OK(cudaEventElapsedTime(&ms, a, b));
  if (ms_out) *ms_out = ms / std::max(iters, 1);
  cudaEventDestroy(a);
  cudaEventDestroy(b);
  return 0;
}
}  // namespace

extern "C" {
#pragma GCC visibility push(default)

const char* prisma_last_error(void) { return get_last_error(); }
const char* prisma_version(void) { return "prisma_b200 0.1 (sm_90a)"; }

int prisma_device_count(void) {
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess) {
    set_last_error(std::string("cudaGetDeviceCount: ") + cudaGetErrorString(e));
    return -2;
  }
  return n;
}

int prisma_depth_create(const char* encoder, int device, prisma_engine** out) {
  API_GUARD_BEGIN
  PRISMA_CHECK(encoder != nullptr && out != nullptr, "null argument");
  DepthEngine* d = new DepthEngine();
  int r = d->init(encoder, device);
  if (r != 0) { delete d; return r; }
  prisma_engine* e = new prisma_engine{1, d, nullptr};
  *out = e;
  return 0;
  API_GUARD_END
}

static DepthEngine* as_depth(prisma_engine* e) {
  if (!e || e->kind != 1 || !e->depth) { set_last_error("not a depth engine handle"); return nullptr; }
  return e->depth;
}

int prisma_depth_load_tensor(prisma_engine* e, const char* name, const float* data, const int64_t* shape, int ndim) {
  API_GUARD_BEGIN
  DepthEngine* d = as_depth(e);
  if (!d) return -1;
  PRISMA_CHECK(name && data && shape && ndim >= 1 && ndim <= 4, "bad tensor");
  return d->load_tensor(name, data, shape, ndim);
  API_GUARD_END
}
int prisma_depth_finalize(prisma_engine* e) {
  API_GUARD_BEGIN
  DepthEngine* d = as_depth(e);
  return d ? d->finalize() : -1;
  API_GUARD_END
}
int prisma_depth_infer(prisma_engine* e, const uint8_t* rgb, int h, int w, float* depth_out, uint8_t* rgb_out,
                       float* min_out, float* max_out) {
  API_GUARD_BEGIN
  DepthEngine* d = as_depth(e);
  return d ? d->infer(rgb, 1, h, w, depth_out, rgb_out, min_out, max_out) : -1;
  API_GUARD_END
}
int prisma_depth_infer_batch(prisma_engine* e, const uint8_t* rgb, int n, int h, int w, float* depth_out,
                             uint8_t* rgb_out, float* min_out, float* max_out) {
  API_GUARD_BEGIN
  DepthEngine* d = as_depth(e);
  return d ? d->infer(rgb, n, h, w, depth_out, rgb_out, min_out, max_out) : -1;
  API_GUARD_END
}
int prisma_depth_infer_stream(prisma_engine* e, const uint8_t* rgb, int n, int h, int w, int pass_frames, float* depth_out,
                              uint8_t* rgb_out, float* min_out, float* max_out) {
  API_GUARD_BEGIN
  DepthEngine* d = as_depth(e);
  return d ? d->infer_stream(rgb, n, h, w, pass_frames, depth_out, rgb_out, min_out, max_out) : -1;
  API_GUARD_END
}
int prisma_host_alloc(size_t bytes, void** out) {
  API_GUARD_BEGIN
  PRISMA_CHECK(out != nullptr && bytes > 0, "bad argument");
  *out = nullptr;
  PRISMA_CUDA_OK(cudaMallocHost(out, bytes));
  return 0;
  API_GUARD_END
}
int prisma_host_free(void* p) {
  API_GUARD_BEGIN
  if (p) PRISMA_CUDA_OK(cudaFreeHost(p));
  return 0;
  API_GUARD_END
}
int prisma_depth_infer_resident(prisma_engine* e, int h, int w, int n, int iters, float* ms_per_iter) {
  API_GUARD_BEGIN
  DepthEngine* d = as_depth(e);
  return d ? d->infer_resident(h, w, n, iters, ms_per_iter) : -1;
  API_GUARD_END
}
int prisma_depth_encode(prisma_engine* e, const float* prediction, int h, int w, int flip, uint8_t* rgb_out,
                        float* min_out, float* max_out) {
  API_GUARD_BEGIN
  DepthEngine* d = as_depth(e);
  PRISMA_CHECK(prediction && rgb_out, "null argument");
  return d ? d->encode(prediction, h, w, flip, rgb_out, min_out, max_out) : -1;
  API_GUARD_END
}
int prisma_depth_encode_png(prisma_engine* e, const float* prediction, int h, int w, int flip, uint8_t* rgb_out,
                            float* min_out, float* max_out) {
  API_GUARD_BEGIN
  DepthEngine* d = as_depth(e);
  PRISMA_CHECK(prediction && rgb_out, "null argument");
  return d ? d->encode(prediction, h, w, flip, rgb_out, min_out, max_out, 1) : -1;
  API_GUARD_END
}
int prisma_depth_infer_image(prisma_engine* e, const uint8_t* rgb, int h, int w, float* depth_out, uint8_t* png_rgb_out,
                             float* min_out, float* max_out) {
  API_GUARD_BEGIN
  DepthEngine* d = as_depth(e);
  return d ? d->infer_image(rgb, h, w, depth_out, png_rgb_out, min_out, max_out) : -1;
  API_GUARD_END
}
long long prisma_depth_read_tap(prisma_engine* e, const char* name, float* out, long long capacity) {
  API_GUARD_BEGIN
  DepthEngine* d = as_depth(e);
  return d ? d->read_tap(name, out, capacity) : -1;
  API_GUARD_END
}
int prisma_depth_profile(prisma_engine* e, int h, int w, int n, float* out8) {
  API_GUARD_BEGIN
  DepthEngine* d = as_depth(e);
  return d ? d->profile(h, w, n, out8) : -1;
  API_GUARD_END
}
int prisma_depth_work(prisma_engine* e, int h, int w, int n, double* out4) {
  API_GUARD_BEGIN
  DepthEngine* d = as_depth(e);
  if (!d) return -1;
  PRISMA_TRY(d->build_plan(h, w, n));
  out4[0] = d->work_linear;
  out4[1] = d->work_attn;
  out4[2] = d->work_head;
  out4[3] = (double)d->steps.size();
  return 0;
  API_GUARD_END
}
int prisma_engine_destroy(prisma_engine* e) {
  API_GUARD_BEGIN
  if (!e) return 0;
  delete e->depth;
  delete e->corr;
  delete e->raft;
  delete e->solo;
  delete e;
  return 0;
  API_GUARD_END
}


int prisma_debug_gemm(int device, const float* A, const float* W, const float* bias, float* Dout, int M, int N, int K,
                      int act, int force_bn, int iters, float* ms_out) {
  API_GUARD_BEGIN
  int sms = 0;
  PRISMA_TRY(device_sms(device, &sms));
  Scratch sc;
  const int Kp = round_up(K, 8);  // row pitch must be a multiple of 16 bytes
  const int Kw = round_up(K, 64), Nw = round_up(N, 256);
  auto hA = to_half_padded(A, M, K, M, Kp);
  auto hW = to_half_padded(W, N, K, Nw, Kw);
  __half* dA = sc.alloc<__half>(hA.size());
  __half* dW = sc.alloc<__half>(hW.size());
  float* dB = sc.alloc<float>(round_up(N, 8));
  float* dD = sc.alloc<float>((size_t)M * N);
  PRISMA_CHECK(dA && dW && dB && dD, "cudaMalloc failed");
  PRISMA_CUDA_OK(cudaMemcpy(dA, hA.data(), hA.size() * 2, cudaMemcpyHostToDevice));
  PRISMA_CUDA_OK(cudaMemcpy(dW, hW.data(), hW.size() * 2, cudaMemcpyHostToDevice));
  if (bias) PRISMA_CUDA_OK(cudaMemcpy(dB, bias, N * 4, cudaMemcpyHostToDevice));
  GemmEpilogue ep;
  ep.bias = bias ? dB : nullptr;
  ep.act = act < 0 ? 0 : act;
  ep.out_f32 = act == -1 ? nullptr : dD;  // act == -1: mainloop only (no stores), act == -2: fp16 output
  ep.out_f32_ld = N;
  __half* dH = nullptr;
  if (act == -2) {
    dH = sc.alloc<__half>((size_t)M * N);
    ep.out_f32 = nullptr;
    ep.out_f16 = dH;
    ep.out_f16_ld = N;
  }
  if (act == -4) {  // TMA-store epilogue (dense fp32, scaled)
    ep.bias = nullptr;
    ep.alpha = 0.0625f;
    ep.tma_store = true;
  }
  if (act == -5) {  // TMA-store epilogue, fp16 destination (scaled): the path of the RAFT correlation volume; N % 8 == 0
    PRISMA_CHECK(N % 8 == 0, "debug gemm: the fp16 TMA-store path needs N % 8 == 0");
    dH = sc.alloc<__half>((size_t)M * N);
    PRISMA_CHECK(dH != nullptr, "cudaMalloc failed");
    PRISMA_CUDA_OK(cudaMemset(dH, 0xFF, (size_t)M * N * 2));  // NaN pattern: every element must be written
    ep.bias = nullptr;
    ep.alpha = 0.0625f;
    ep.out_f32 = nullptr;
    ep.out_f16 = dH;
    ep.out_f16_ld = N;
    ep.tma_store = true;
  }
  if (act == -6 || act == -7) {  // TMA-store epilogue, fp16 destination with bias + GELU (-6) / ReLU (-7): the ViT qkv / fc1 path
    PRISMA_CHECK(N % 8 == 0, "debug gemm: the fp16 TMA-store path needs N % 8 == 0");
    dH = sc.alloc<__half>((size_t)M * N);
    PRISMA_CHECK(dH != nullptr, "cudaMalloc failed");
    PRISMA_CUDA_OK(cudaMemset(dH, 0xFF, (size_t)M * N * 2));
    ep.act = act == -6 ? 1 : 2;
    ep.out_f32 = nullptr;
    ep.out_f16 = dH;
    ep.out_f16_ld = N;
    ep.tma_store = true;
  }
  if (act == -8) {  // in-place fp32 residual through the TMA reduce-add epilogue: D (zeros) += acc + bias, once per launch
    ep.res_f32 = dD;
    ep.res_f32_ld = N;
    ep.tma_store = true;
    PRISMA_CUDA_OK(cudaMemset(dD, 0, (size_t)M * N * 4));
  }
  if (act == -3) {  // micro-benchmark of the residual-stream epilogue: D += acc in place (fp32 read + write)
    ep.res_f32 = dD;
    ep.res_f32_ld = N;
    PRISMA_CUDA_OK(cudaMemset(dD, 0, (size_t)M * N * 4));
  }
  GemmLaunch g;
  const int off[1] = {0};
  PRISMA_TRY(gemm_prepare(&g, dA, M, K, Kp, dW, Nw, M, N, 1, off, ep, sms, force_bn));
  PRISMA_TRY(timed(0, iters > 0 ? iters : 1, ms_out, [&]() { return gemm_run(g, 0); }));
  if (act == -5 || act == -6 || act == -7) {
    std::vector<__half> hd((size_t)M * N);
    PRISMA_CUDA_OK(cudaMemcpy(hd.data(), dH, hd.size() * 2, cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < hd.size(); ++i) Dout[i] = __half2float(hd[i]);
    return 0;
  }
  PRISMA_CUDA_OK(cudaMemcpy(Dout, dD, (size_t)M * N * 4, cudaMemcpyDeviceToHost));
  return 0;
  API_GUARD_END
}

// D = A[M,K] * W[N,K]^T + bias through the 3xTF32 path (fp32-class products on the tensor cores): the operands are split on
// the host into [hi | lo] / [hi | hi | lo] as gemm_prepare_tf32x3 expects.  K is padded to a multiple of 32.
int prisma_debug_gemm_tf32x3(int device, const float* A, const float* W, const float* bias, float* Dout, int M, int N, int K,
                             int force_bn, int iters, float* ms_out) {
  API_GUARD_BEGIN
  int sms = 0;
  PRISMA_TRY(device_sms(device, &sms));
  Scratch sc;
  const int C = round_up(K, 32), Nw = round_up(N, 256);
  auto hi_of = [](float v) { uint32_t u; memcpy(&u, &v, 4); u &= 0xFFFFE000u; float h; memcpy(&h, &u, 4); return h; };
  std::vector<float> hA((size_t)M * 2 * C, 0.f), hW((size_t)Nw * 3 * C, 0.f);
  for (int m = 0; m < M; ++m)
    for (int k = 0; k < K; ++k) {
      const float v = A[(size_t)m * K + k], h = hi_of(v);
      hA[(size_t)m * 2 * C + k] = h;
      hA[(size_t)m * 2 * C + C + k] = v - h;
    }
  for (int n = 0; n < N; ++n)
    for (int k = 0; k < K; ++k) {
      const float v = W[(size_t)n * K + k], h = hi_of(v);
      hW[(size_t)n * 3 * C + k] = h;
      hW[(size_t)n * 3 * C + C + k] = h;
      hW[(size_t)n * 3 * C + 2 * C + k] = v - h;
    }
  float* dA = sc.alloc<float>(hA.size());
  float* dW = sc.alloc<float>(hW.size());
  float* dB = sc.alloc<float>(round_up(N, 8));
  float* dD = sc.alloc<float>((size_t)M * N);
  PRISMA_CHECK(dA && dW && dB && dD, "cudaMalloc failed");
  PRISMA_CUDA_OK(cudaMemcpy(dA, hA.data(), hA.size() * 4, cudaMemcpyHostToDevice));
  PRISMA_CUDA_OK(cudaMemcpy(dW, hW.data(), hW.size() * 4, cudaMemcpyHostToDevice));
  if (bias) PRISMA_CUDA_OK(cudaMemcpy(dB, bias, N * 4, cudaMemcpyHostToDevice));
  GemmEpilogue ep;
  ep.bias = bias ? dB : nullptr;
  ep.out_f32 = dD;
  ep.out_f32_ld = N;
  GemmLaunch g;
  const int off[1] = {0};
  PRISMA_TRY(gemm_prepare_tf32x3(&g, dA, M, C, C, dW, Nw, M, N, 1, off, ep, sms, force_bn));
  PRISMA_TRY(timed(0, iters > 0 ? iters : 1, ms_out, [&]() { return gemm_run(g, 0); }));
  PRISMA_CUDA_OK(cudaMemcpy(Dout, dD, (size_t)M * N * 4, cudaMemcpyDeviceToHost));
  return 0;
  API_GUARD_END
}

int prisma_debug_conv(int device, const float* x, const float* w_oihw, const float* bias, float* y, int H, int W,
                      int Cin, int Cout, int kh, int kw, int relu, float* ms_out) {
  API_GUARD_BEGIN
  int sms = 0;
  PRISMA_TRY(device_sms(device, &sms));
  PRISMA_CHECK(Cin % 8 == 0 && Cout % 8 == 0, "conv: channels must be multiples of 8");
  PRISMA_CHECK(kh * kw <= GEMM_MAX_TAPS && (kh & 1) && (kw & 1), "conv: odd kernel up to 7x7");
  Scratch sc;
  const int ph = kh / 2, pw = kw / 2;  // 'same' padding; the border must be at least that wide
  const int Hp = H + 2 * ph, Wp = W + 2 * pw;
  std::vector<__half> hx((size_t)Hp * Wp * Cin, __float2half_rn(0.f));
  for (int yy = 0; yy < H; ++yy)
    for (int xx = 0; xx < W; ++xx)
      for (int c = 0; c < Cin; ++c)
        hx[((size_t)(yy + ph) * Wp + xx + pw) * Cin + c] = __float2half_rn(x[((size_t)yy * W + xx) * Cin + c]);
  const int kc = ceil_div(Cin, 64), taps = kh * kw, Kw = taps * kc * 64, Nw = round_up(Cout, 256);
  std::vector<__half> hw((size_t)Nw * Kw, __float2half_rn(0.f));
  for (int n = 0; n < Cout; ++n)
    for (int t = 0; t < taps; ++t)
      for (int c = 0; c < Cin; ++c)
        hw[(size_t)n * Kw + (size_t)t * kc * 64 + c] = __float2half_rn(w_oihw[((size_t)n * Cin + c) * taps + t]);
  __half* dx = sc.alloc<__half>(hx.size());
  __half* dw = sc.alloc<__half>(hw.size());
  float* db = sc.alloc<float>(round_up(Cout, 8));
  float* dy = sc.alloc<float>((size_t)Hp * Wp * Cout);
  PRISMA_CHECK(dx && dw && db && dy, "cudaMalloc failed");
  PRISMA_CUDA_OK(cudaMemcpy(dx, hx.data(), hx.size() * 2, cudaMemcpyHostToDevice));
  PRISMA_CUDA_OK(cudaMemcpy(dw, hw.data(), hw.size() * 2, cudaMemcpyHostToDevice));
  if (bias) PRISMA_CUDA_OK(cudaMemcpy(db, bias, Cout * 4, cudaMemcpyHostToDevice));
  int off[GEMM_MAX_TAPS];
  for (int ky = 0; ky < kh; ++ky)
    for (int kx = 0; kx < kw; ++kx) off[ky * kw + kx] = (ky - ph) * Wp + (kx - pw);
  GemmEpilogue ep;
  ep.bias = bias ? db : nullptr;
  ep.act = relu ? 2 : 0;
  ep.out_f32 = dy;
  ep.out_f32_ld = Cout;
  // generic border width: use LINEAR mapping and crop on the host (the engine's 3x3 path uses ROW_PADDED)
  GemmLaunch g;
  PRISMA_TRY(gemm_prepare(&g, dx, (long long)Hp * Wp, Cin, Cin, dw, Nw, Hp * Wp, Cout, taps, off, ep, sms, 0));
  PRISMA_TRY(timed(0, 1, ms_out, [&]() { return gemm_run(g, 0); }));
  std::vector<float> hy((size_t)Hp * Wp * Cout);
  PRISMA_CUDA_OK(cudaMemcpy(hy.data(), dy, hy.size() * 4, cudaMemcpyDeviceToHost));
  for (int yy = 0; yy < H; ++yy)
    for (int xx = 0; xx < W; ++xx)
      memcpy(y + ((size_t)yy * W + xx) * Cout, hy.data() + ((size_t)(yy + ph) * Wp + xx + pw) * Cout, Cout * 4);
  return 0;
  API_GUARD_END
}

int prisma_debug_attention(int device, const float* qkv, float* out, int T, int heads, int iters, float* ms_out) {
  API_GUARD_BEGIN
  int sms = 0;
  PRISMA_TRY(device_sms(device, &sms));
  const int D = heads * 64;
  Scratch sc;
  std::vector<__half> h((size_t)T * 3 * D);
  for (int t = 0; t < T; ++t)
    for (int c = 0; c < 3 * D; ++c)
      h[(size_t)t * 3 * D + c] = __float2half_rn(qkv[(size_t)t * 3 * D + c] * (c < D ? 0.125f : 1.f));
  __half* dq = sc.alloc<__half>(h.size());
  __half* dO = sc.alloc<__half>((size_t)T * D);
  PRISMA_CHECK(dq && dO, "cudaMalloc failed");
  PRISMA_CUDA_OK(cudaMemcpy(dq, h.data(), h.size() * 2, cudaMemcpyHostToDevice));
  AttnLaunch a;
  PRISMA_TRY(attention_prepare(&a, dq, dO, 1, T, heads, D));
  PRISMA_TRY(timed(0, iters > 0 ? iters : 1, ms_out, [&]() { return attention_run(a, 0); }));
  std::vector<__half> ho((size_t)T * D);
  PRISMA_CUDA_OK(cudaMemcpy(ho.data(), dO, ho.size() * 2, cudaMemcpyDeviceToHost));
  for (size_t i = 0; i < ho.size(); ++i) out[i] = __half2float(ho[i]);
  return 0;
  API_GUARD_END
}

int prisma_debug_layernorm(int device, const float* x, const float* g, const float* b, float* y, int rows, int D) {
  API_GUARD_BEGIN
  int sms = 0;
  PRISMA_TRY(device_sms(device, &sms));
  Scratch sc;
  float* dx = sc.alloc<float>((size_t)rows * D);
  float* dg = sc.alloc<float>(D);
  float* db = sc.alloc<float>(D);
  __half* dy = sc.alloc<__half>((size_t)rows * D);
  PRISMA_CHECK(dx && dg && db && dy, "cudaMalloc failed");
  PRISMA_CUDA_OK(cudaMemcpy(dx, x, (size_t)rows * D * 4, cudaMemcpyHostToDevice));
  PRISMA_CUDA_OK(cudaMemcpy(dg, g, D * 4, cudaMemcpyHostToDevice));
  PRISMA_CUDA_OK(cudaMemcpy(db, b, D * 4, cudaMemcpyHostToDevice));
  PRISMA_TRY(layernorm_f16(dx, dg, db, dy, rows, D, 1e-6f, 0));
  std::vector<__half> hy((size_t)rows * D);
  PRISMA_CUDA_OK(cudaMemcpy(hy.data(), dy, hy.size() * 2, cudaMemcpyDeviceToHost));
  for (size_t i = 0; i < hy.size(); ++i) y[i] = __half2float(hy[i]);
  return 0;
  API_GUARD_END
}

int prisma_debug_da_preprocess(int device, const uint8_t* rgb, int h, int w, float* out, int hn, int wn) {
  API_GUARD_BEGIN
  int sms = 0;
  PRISMA_TRY(device_sms(device, &sms));
  int ewn, ehn;
  da_net_size(w, h, &ewn, &ehn);
  PRISMA_CHECK(ewn == wn && ehn == hn, "net size mismatch: expected " + std::to_string(ewn) + "x" + std::to_string(ehn));
  Scratch sc;
  uint8_t* di = sc.alloc<uint8_t>((size_t)h * w * 3);
  float* dout = sc.alloc<float>((size_t)3 * hn * wn);
  PRISMA_CHECK(di && dout, "cudaMalloc failed");
  PRISMA_CUDA_OK(cudaMemcpy(di, rgb, (size_t)h * w * 3, cudaMemcpyHostToDevice));
  PRISMA_TRY(da_preprocess(di, h, w, dout, hn, wn, 0));
  PRISMA_CUDA_OK(cudaMemcpy(out, dout, (size_t)3 * hn * wn * 4, cudaMemcpyDeviceToHost));
  return 0;
  API_GUARD_END
}

// ------------------------------------------------------------------------------------------------ RAFT band (HBM-bound stages)
static FlowCorr* as_corr(prisma_engine* e) {
  if (!e || e->kind != 2 || !e->corr) { set_last_error("not a flow-correlation handle"); return nullptr; }
  return e->corr;
}

int prisma_flow_preprocess(int device, const uint8_t* rgb, int h, int w, double scale, uint8_t* resized, float* chw) {
  API_GUARD_BEGIN
  int sms = 0;
  PRISMA_TRY(device_sms(device, &sms));
  PRISMA_CHECK(rgb && chw && h > 0 && w > 0 && scale > 0.0, "bad argument");
  const int hs = (int)nearbyint((double)h * scale), ws = (int)nearbyint((double)w * scale);
  const int pad_h = (((hs / 8) + 1) * 8 - hs) % 8, pad_w = (((ws / 8) + 1) * 8 - ws) % 8;  // common/flow.py:46-53
  const int pad[4] = {pad_w / 2, pad_w - pad_w / 2, pad_h / 2, pad_h - pad_h / 2};
  const int hp = hs + pad_h, wp = ws + pad_w;
  Scratch sc;
  uint8_t* di = sc.alloc<uint8_t>((size_t)h * w * 3);
  uint8_t* dr = sc.alloc<uint8_t>((size_t)hs * ws * 3);
  float* dc = sc.alloc<float>((size_t)3 * hp * wp);
  PRISMA_CHECK(di && dr && dc, "cudaMalloc failed");
  PRISMA_CUDA_OK(cudaMemcpy(di, rgb, (size_t)h * w * 3, cudaMemcpyHostToDevice));
  PRISMA_TRY(raft_preprocess(di, h, w, hs, ws, scale, pad, dr, dc, 0));
  if (resized) PRISMA_CUDA_OK(cudaMemcpy(resized, dr, (size_t)hs * ws * 3, cudaMemcpyDeviceToHost));
  PRISMA_CUDA_OK(cudaMemcpy(chw, dc, (size_t)3 * hp * wp * 4, cudaMemcpyDeviceToHost));
  return 0;
  API_GUARD_END
}

int prisma_flow_encode(int device, const float* flow, int h, int w, uint8_t* rgb_out, float* max_disp_out) {
  API_GUARD_BEGIN
  int sms = 0;
  PRISMA_TRY(device_sms(device, &sms));
  PRISMA_CHECK(flow && rgb_out, "null argument");
  Scratch sc;
  float* df = sc.alloc<float>((size_t)h * w * 2);
  uint8_t* dr = sc.alloc<uint8_t>((size_t)h * w * 3);
  uint32_t* dm = sc.alloc<uint32_t>(2);
  float* dmax = sc.alloc<float>(2);
  PRISMA_CHECK(df && dr && dm && dmax, "cudaMalloc failed");
  PRISMA_CUDA_OK(cudaMemcpy(df, flow, (size_t)h * w * 8, cudaMemcpyHostToDevice));
  PRISMA_TRY(flow_encode(df, h, w, dr, dm, dmax, sms, 0));
  PRISMA_CUDA_OK(cudaMemcpy(rgb_out, dr, (size_t)h * w * 3, cudaMemcpyDeviceToHost));
  float m = 0;
  PRISMA_CUDA_OK(cudaMemcpy(&m, dmax, 4, cudaMemcpyDeviceToHost));
  if (max_disp_out) *max_disp_out = m;
  return 0;
  API_GUARD_END
}

int prisma_flow_masks(int device, const float* fwd, const float* bwd, int h, int w, uint8_t* fwd_mask, uint8_t* bwd_mask,
                      uint16_t* fwd_u16, uint16_t* bwd_u16) {
  API_GUARD_BEGIN
  int sms = 0;
  PRISMA_TRY(device_sms(device, &sms));
  PRISMA_CHECK(fwd && bwd && fwd_mask && bwd_mask, "null argument");
  Scratch sc;
  const size_t n = (size_t)h * w;
  float* df = sc.alloc<float>(n * 2);
  float* db = sc.alloc<float>(n * 2);
  uint8_t* mf = sc.alloc<uint8_t>(n);
  uint8_t* mb = sc.alloc<uint8_t>(n);
  uint16_t* uf = sc.alloc<uint16_t>(n * 3);
  uint16_t* ub = sc.alloc<uint16_t>(n * 3);
  PRISMA_CHECK(df && db && mf && mb && uf && ub, "cudaMalloc failed");
  PRISMA_CUDA_OK(cudaMemcpy(df, fwd, n * 8, cudaMemcpyHostToDevice));
  PRISMA_CUDA_OK(cudaMemcpy(db, bwd, n * 8, cudaMemcpyHostToDevice));
  PRISMA_TRY(flow_consistency_masks(df, db, h, w, mf, mb, sms, 0));
  PRISMA_TRY(flow_encode_u16(df, mf, h, w, uf, sms, 0));
  PRISMA_TRY(flow_encode_u16(db, mb, h, w, ub, sms, 0));
  PRISMA_CUDA_OK(cudaMemcpy(fwd_mask, mf, n, cudaMemcpyDeviceToHost));
  PRISMA_CUDA_OK(cudaMemcpy(bwd_mask, mb, n, cudaMemcpyDeviceToHost));
  if (fwd_u16) PRISMA_CUDA_OK(cudaMemcpy(fwd_u16, uf, n * 6, cudaMemcpyDeviceToHost));
  if (bwd_u16) PRISMA_CUDA_OK(cudaMemcpy(bwd_u16, ub, n * 6, cudaMemcpyDeviceToHost));
  return 0;
  API_GUARD_END
}

int prisma_flowcorr_create(int device, int batch, int h8, int w8, prisma_engine** out) {
  API_GUARD_BEGIN
  PRISMA_CHECK(out != nullptr, "null argument");
  FlowCorr* c = new FlowCorr();
  int r = c->init(device, batch, h8, w8);
  if (r != 0) { delete c; return r; }
  *out = new prisma_engine{2, nullptr, c};
  return 0;
  API_GUARD_END
}
int prisma_flowcorr_set_fmaps(prisma_engine* e, const float* fmap1, const float* fmap2) {
  API_GUARD_BEGIN
  FlowCorr* c = as_corr(e);
  PRISMA_CHECK(fmap1 && fmap2, "null argument");
  return c ? c->set_fmaps(fmap1, fmap2) : -1;
  API_GUARD_END
}
int prisma_flowcorr_build(prisma_engine* e, int iters, float* ms_out) {
  API_GUARD_BEGIN
  FlowCorr* c = as_corr(e);
  return c ? c->time_build(iters > 0 ? iters : 1, ms_out) : -1;
  API_GUARD_END
}
int prisma_flowcorr_lookup(prisma_engine* e, const float* coords, float* out, int iters, float* ms_out) {
  API_GUARD_BEGIN
  FlowCorr* c = as_corr(e);
  PRISMA_CHECK(coords != nullptr, "null argument");
  return c ? c->lookup_host(coords, out, iters > 0 ? iters : 1, ms_out) : -1;
  API_GUARD_END
}
int prisma_flowcorr_read_level(prisma_engine* e, int level, int b, int row0, int nrows, float* out) {
  API_GUARD_BEGIN
  FlowCorr* c = as_corr(e);
  return c ? c->read_level(level, b, row0, nrows, out) : -1;
  API_GUARD_END
}
int prisma_flowcorr_work(prisma_engine* e, double* out2) {
  API_GUARD_BEGIN
  FlowCorr* c = as_corr(e);
  if (!c) return -1;
  out2[0] = c->flops_build;
  out2[1] = c->bytes_build;
  return 0;
  API_GUARD_END
}

// ------------------------------------------------------------------------------------------------ RAFT engine
static RaftEngine* as_raft(prisma_engine* e) {
  if (!e || e->kind != 3 || !e->raft) { set_last_error("not a RAFT engine handle"); return nullptr; }
  return e->raft;
}
static SoloEngine* as_solo(prisma_engine* e) {
  if (!e || e->kind != 4 || !e->solo) { set_last_error("not a mask (SOLOv2) engine handle"); return nullptr; }
  return e->solo;
}
int prisma_mask_create(const char* variant, int device, prisma_engine** out) {
  API_GUARD_BEGIN
  PRISMA_CHECK(out != nullptr && variant != nullptr, "null argument");
  SoloEngine* m = new SoloEngine();
  int rc = m->init(variant, device);
  if (rc != 0) { delete m; return rc; }
  prisma_engine* e = new prisma_engine{4, nullptr, nullptr};
  e->solo = m;
  *out = e;
  return 0;
  API_GUARD_END
}
int prisma_mask_load_tensor(prisma_engine* e, const char* name, const float* data, const int64_t* shape, int ndim) {
  API_GUARD_BEGIN
  SoloEngine* m = as_solo(e);
  if (!m) return -1;
  PRISMA_CHECK(name && data && shape && ndim >= 1 && ndim <= 4, "bad tensor");
  return m->load_tensor(name, data, shape, ndim);
  API_GUARD_END
}
int prisma_mask_finalize(prisma_engine* e) {
  API_GUARD_BEGIN
  SoloEngine* m = as_solo(e);
  return m ? m->finalize() : -1;
  API_GUARD_END
}
int prisma_mask_infer(prisma_engine* e, const uint8_t* rgb, int h, int w, float confidence, uint8_t* union_mask, int* n_inst,
                      float* scores, int32_t* labels, uint8_t* inst_masks, float* ms_out) {
  API_GUARD_BEGIN
  SoloEngine* m = as_solo(e);
  return m ? m->infer(rgb, h, w, confidence, union_mask, n_inst, scores, labels, inst_masks, ms_out) : -1;
  API_GUARD_END
}
int prisma_mask_inject_feat(prisma_engine* e, int level, const float* nchw, int h, int w) {
  API_GUARD_BEGIN
  SoloEngine* m = as_solo(e);
  PRISMA_CHECK(nchw != nullptr, "null argument");
  return m ? m->inject_feat(level, nchw, h, w) : -1;
  API_GUARD_END
}
int prisma_mask_infer_from_feats(prisma_engine* e, int h, int w, int img_h, int img_w, float confidence, uint8_t* union_mask,
                                 int* n_inst, float* scores, int32_t* labels, uint8_t* inst_masks) {
  API_GUARD_BEGIN
  SoloEngine* m = as_solo(e);
  return m ? m->infer_from_feats(h, w, img_h, img_w, confidence, union_mask, n_inst, scores, labels, inst_masks) : -1;
  API_GUARD_END
}
long long prisma_mask_read_tap(prisma_engine* e, const char* name, float* out, long long capacity) {
  API_GUARD_BEGIN
  SoloEngine* m = as_solo(e);
  return m ? m->read_tap(name, out, capacity) : -1;
  API_GUARD_END
}
// network-input size arithmetic of each band's transform (host logic only: no GPU needed)
int prisma_net_size(const char* band, int w, int h, int* wn, int* hn) {
  API_GUARD_BEGIN
  PRISMA_CHECK(band && wn && hn && w > 0 && h > 0, "bad argument");
  const std::string b(band);
  if (b == "depth_anything") da_net_size(w, h, wn, hn);
  else if (b == "depth_midas") midas_net_size(w, h, wn, hn);
  else if (b == "depth_anything_metric") { *wn = 518; *hn = 392; }
  else if (b == "mask_mmdet") {
    SoloEngine e;  // only its size rule is used
    int nh, nw, hp, wp;
    e.net_shape(h, w, &nh, &nw, &hp, &wp);
    *wn = nw; *hn = nh;
  } else { set_last_error("unknown band '" + b + "'"); return -1; }
  return 0;
  API_GUARD_END
}
int prisma_mask_sdf(int device, const uint8_t* union_mask, int h, int w, uint8_t* green_out) {
  API_GUARD_BEGIN
  int sms = 0;
  PRISMA_TRY(device_sms(device, &sms));
  PRISMA_CHECK(union_mask && green_out && h > 0 && w > 0 && w <= 3000, "bad argument (frames up to 3000 pixels wide)");
  Scratch sc;
  const size_t n = (size_t)h * w;
  uint8_t* dm = sc.alloc<uint8_t>(n);
  uint8_t* dg = sc.alloc<uint8_t>(n);
  int* ds = sc.alloc<int>(2 * n);
  PRISMA_CHECK(dm && dg && ds, "cudaMalloc failed");
  PRISMA_CUDA_OK(cudaMemcpy(dm, union_mask, n, cudaMemcpyHostToDevice));
  PRISMA_TRY(mask_sdf_green(dm, h, w, ds, dg, 0));
  PRISMA_CUDA_OK(cudaMemcpy(green_out, dg, n, cudaMemcpyDeviceToHost));
  return 0;
  API_GUARD_END
}
int prisma_mask_work(prisma_engine* e, int h, int w, double* out8) {
  API_GUARD_BEGIN
  SoloEngine* m = as_solo(e);
  if (!m) return -1;
  PRISMA_CHECK(out8 != nullptr, "null argument");
  int nh, nw, hp, wp;
  m->net_shape(h, w, &nh, &nw, &hp, &wp);
  out8[0] = m->flops; out8[1] = m->launches; out8[2] = nh; out8[3] = nw; out8[4] = hp; out8[5] = wp; out8[6] = 0; out8[7] = 0;
  return 0;
  API_GUARD_END
}

int prisma_flow_create(int device, prisma_engine** out) {
  API_GUARD_BEGIN
  PRISMA_CHECK(out != nullptr, "null argument");
  RaftEngine* r = new RaftEngine();
  int rc = r->init(device);
  if (rc != 0) { delete r; return rc; }
  prisma_engine* e = new prisma_engine{3, nullptr, nullptr};
  e->raft = r;
  *out = e;
  return 0;
  API_GUARD_END
}
int prisma_flow_load_tensor(prisma_engine* e, const char* name, const float* data, const int64_t* shape, int ndim) {
  API_GUARD_BEGIN
  RaftEngine* r = as_raft(e);
  if (!r) return -1;
  PRISMA_CHECK(name && data && shape && ndim >= 1 && ndim <= 4, "bad tensor");
  return r->load_tensor(name, data, shape, ndim);
  API_GUARD_END
}
int prisma_flow_finalize(prisma_engine* e) {
  API_GUARD_BEGIN
  RaftEngine* r = as_raft(e);
  return r ? r->finalize() : -1;
  API_GUARD_END
}
int prisma_flow_infer(prisma_engine* e, const uint8_t* prev, const uint8_t* curr, int h, int w, double scale, int iters,
                      float* fwd, float* bwd, uint8_t* fwd_rgb, uint8_t* bwd_rgb, float* max_fwd, float* max_bwd,
                      float* ms_out) {
  API_GUARD_BEGIN
  RaftEngine* r = as_raft(e);
  return r ? r->infer(prev, curr, h, w, scale, iters, fwd, bwd, fwd_rgb, bwd_rgb, max_fwd, max_bwd, ms_out) : -1;
  API_GUARD_END
}
int prisma_flow_infer_video(prisma_engine* e, const uint8_t* prev, const uint8_t* curr, int h, int w, double scale, int iters,
                            int reuse_prev, float* fwd, float* bwd, uint8_t* fwd_rgb, uint8_t* bwd_rgb, float* max_fwd,
                            float* max_bwd, float* ms_out) {
  API_GUARD_BEGIN
  RaftEngine* r = as_raft(e);
  return r ? r->infer(prev, curr, h, w, scale, iters, fwd, bwd, fwd_rgb, bwd_rgb, max_fwd, max_bwd, ms_out, reuse_prev) : -1;
  API_GUARD_END
}
int prisma_flow_infer_stream(prisma_engine* e, const uint8_t* frames, int n, int h, int w, double scale, int iters,
                             int continue_clip, float* fwd, float* bwd, uint8_t* fwd_rgb, uint8_t* bwd_rgb, float* max_fwd,
                             float* max_bwd, int* pairs_out) {
  API_GUARD_BEGIN
  RaftEngine* r = as_raft(e);
  return r ? r->infer_stream(frames, n, h, w, scale, iters, continue_clip, fwd, bwd, fwd_rgb, bwd_rgb, max_fwd, max_bwd, pairs_out) : -1;
  API_GUARD_END
}
int prisma_flow_infer_resident(prisma_engine* e, int h, int w, double scale, int iters, int reps, float* ms_per_pass) {
  API_GUARD_BEGIN
  RaftEngine* r = as_raft(e);
  return r ? r->time_resident(h, w, scale, iters, reps, ms_per_pass) : -1;
  API_GUARD_END
}
long long prisma_flow_read_tap(prisma_engine* e, const char* name, float* out, long long capacity) {
  API_GUARD_BEGIN
  RaftEngine* r = as_raft(e);
  return r ? r->read_tap(name, out, capacity) : -1;
  API_GUARD_END
}
int prisma_flow_work(prisma_engine* e, int h, int w, double scale, int iters, double* out4) {
  API_GUARD_BEGIN
  RaftEngine* r = as_raft(e);
  if (!r) return -1;
  r->use_pairs(1);
  PRISMA_TRY(r->build_plan(h, w, scale, iters));
  int full_steps = 0;
  for (const auto& st : r->steps) full_steps += (st.group & 1) ? 1 : 0;  // steps of the full pass (the video pass has fewer)
  out4[0] = r->flops; out4[1] = (double)full_steps; out4[2] = r->Hs; out4[3] = r->Ws;
  return 0;
  API_GUARD_END
}
int prisma_flow_work_detail(prisma_engine* e, int h, int w, double scale, int iters, double* out8) {
  API_GUARD_BEGIN
  RaftEngine* r = as_raft(e);
  if (!r) return -1;
  PRISMA_CHECK(out8 != nullptr, "null argument");
  r->use_pairs(r->clip_pairs(h, w, scale));
  PRISMA_TRY(r->build_plan(h, w, scale, iters));
  int full_steps = 0, video_steps = 0;
  for (const auto& st : r->steps) { full_steps += (st.group & 1) ? 1 : 0; video_steps += (st.group & 2) ? 1 : 0; }
  out8[0] = r->flops_conv; out8[1] = r->flops_conv_video;
  out8[2] = r->corr_block()->flops_build; out8[3] = r->corr_block()->bytes_build;
  out8[4] = full_steps; out8[5] = video_steps; out8[6] = r->Hs; out8[7] = r->Ws;
  return 0;
  API_GUARD_END
}
int prisma_flow_set_pairs_per_pass(prisma_engine* e, int pairs) {
  API_GUARD_BEGIN
  RaftEngine* r = as_raft(e);
  return r ? r->set_pairs_per_pass(pairs) : -1;
  API_GUARD_END
}
int prisma_flow_pairs_per_pass(prisma_engine* e) {
  API_GUARD_BEGIN
  RaftEngine* r = as_raft(e);
  return r ? r->pairs_per_pass() : -1;
  API_GUARD_END
}
int prisma_flow_plan_pairs(prisma_engine* e) {
  API_GUARD_BEGIN
  RaftEngine* r = as_raft(e);
  return r ? r->plan_pairs() : -1;
  API_GUARD_END
}
int prisma_flow_profile(prisma_engine* e, int h, int w, double scale, int iters, float* out8) {
  API_GUARD_BEGIN
  RaftEngine* r = as_raft(e);
  PRISMA_CHECK(out8 != nullptr, "null argument");
  return r ? r->profile(h, w, scale, iters, out8) : -1;
  API_GUARD_END
}

#pragma GCC visibility pop
}  // extern "C"
