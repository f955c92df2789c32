// prisma_b200 -- host side of the wgmma shifted-row GEMM: TMA descriptor encode, tile-shape choice, launch.
#include "gemm_tc.cuh"

#include <atomic>
#include <mutex>

#include <nvtx3/nvToolsExt.h>

namespace prisma {

NvtxRange::NvtxRange(const char* name) { nvtxRangePushA(name); }
NvtxRange::~NvtxRange() { nvtxRangePop(); }

// Programmatic dependent launch is OFF unless PRISMA_PDL=1: the ~330 kernels of a RAFT pass are already back to back inside
// a CUDA graph, and tests/test_raft_gpu.py has seen a wrong max displacement under it (an ordering it must not change).
// Kept only as an experiment switch.
bool pdl_enabled() {
  static const bool on = [] { const char* e = getenv("PRISMA_PDL"); return e && e[0] == '1'; }();
  return on;
}

int device_sm_count() {
  static std::atomic<int> cache[64] = {};  // engines on several threads (mask lanes) query it concurrently
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  int n = cache[dev].load(std::memory_order_relaxed);
  if (n == 0) {
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) return 132;
    cache[dev].store(n, std::memory_order_relaxed);
  }
  return n;
}

static thread_local std::string g_last_error;
void set_last_error(const std::string& msg) { g_last_error = msg; }
const char* get_last_error() { return g_last_error.c_str(); }

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

int make_tmap_2d_f16(CUtensorMap* out, const void* base, uint64_t cols, uint64_t rows, uint64_t pitch_elems,
                     uint32_t box_cols, uint32_t box_rows) {
  EncodeTiledFn fn = get_encode_fn();
  PRISMA_CHECK(fn != nullptr, "cuTensorMapEncodeTiled entry point not available (no CUDA driver?)");
  PRISMA_CHECK((reinterpret_cast<uintptr_t>(base) & 15) == 0, "TMA base must be 16-byte aligned");
  PRISMA_CHECK((pitch_elems * 2) % 16 == 0, "TMA row pitch must be a multiple of 16 bytes");
  PRISMA_CHECK(box_cols * 2 == 128 && box_rows >= 1 && box_rows <= 256, "TMA box must be 64 fp16 wide, <=256 rows");
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {pitch_elems * 2};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  PRISMA_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed (code " + std::to_string((int)r) + ")");
  return 0;
}

int make_tmap_2d_f32(CUtensorMap* out, const void* base, uint64_t cols, uint64_t rows, uint64_t pitch_elems,
                     uint32_t box_cols, uint32_t box_rows) {
  EncodeTiledFn fn = get_encode_fn();
  PRISMA_CHECK(fn != nullptr, "cuTensorMapEncodeTiled entry point not available (no CUDA driver?)");
  PRISMA_CHECK((reinterpret_cast<uintptr_t>(base) & 15) == 0, "TMA base must be 16-byte aligned");
  PRISMA_CHECK((pitch_elems * 4) % 16 == 0, "TMA row pitch must be a multiple of 16 bytes");
  PRISMA_CHECK(box_cols * 4 == 128 && box_rows >= 1 && box_rows <= 256, "TMA box must be 32 fp32 wide, <=256 rows");
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {pitch_elems * 4};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  PRISMA_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled (fp32) failed (code " + std::to_string((int)r) + ")");
  return 0;
}

// fp16 destination of the TMA-store epilogue: boxes of 32 rows x 64 columns (128-byte rows), 128-byte swizzle
static int make_tmap_2d_f16_store(CUtensorMap* out, const void* base, uint64_t cols, uint64_t rows, uint64_t pitch_elems) {
  EncodeTiledFn fn = get_encode_fn();
  PRISMA_CHECK(fn != nullptr, "cuTensorMapEncodeTiled entry point not available (no CUDA driver?)");
  PRISMA_CHECK((reinterpret_cast<uintptr_t>(base) & 15) == 0, "TMA base must be 16-byte aligned");
  PRISMA_CHECK((pitch_elems * 2) % 16 == 0, "TMA row pitch must be a multiple of 16 bytes");
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {pitch_elems * 2};
  cuuint32_t box[2] = {64, 32};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  PRISMA_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled (fp16 store) failed (code " + std::to_string((int)r) + ")");
  return 0;
}

// Tile-N choice: minimise waves x per-tile time.  The per-tile cost is taken proportional to the operand bytes a tile
// streams per K block ((128 + BN) rows of 128 B) plus the accumulator drain (BN), a model, not a measurement: wide
// tiles move fewer operand bytes per FLOP, narrow ones waste less on padding and fill the last wave better.
int gemm_pick_bn(int M, int N, int num_sms) {
  const int cands[4] = {256, 128, 64, 32};
  int best = 128;
  double best_cost = 1e30;
  const int tiles_m = ceil_div(M, GEMM_BM);
  for (int i = 0; i < 4; ++i) {
    const int bn = cands[i];
    if (bn > 32 && bn >= 2 * round_up(N, 32)) continue;  // mostly padding
    const int tiles = tiles_m * ceil_div(N, bn);
    const int waves = ceil_div(tiles, num_sms);
    const double cost = waves * (double)(GEMM_BM + 2 * bn);
    if (cost < best_cost) { best_cost = cost; best = bn; }
  }
  return best;
}

static int gemm_prepare_impl(GemmLaunch* out, const void* A, long long a_rows, int a_cols, int a_pitch, const void* W,
                             int w_rows, int M, int N, int taps, const int* tap_off, const int* tap_acol, const GemmEpilogue& ep,
                             int num_sms, int force_bn, bool tf32);

int gemm_prepare(GemmLaunch* out, const __half* A, long long a_rows, int a_cols, int a_pitch, const __half* W,
                 int w_rows, int M, int N, int taps, const int* tap_off, const GemmEpilogue& ep, int num_sms,
                 int force_bn) {
  return gemm_prepare_impl(out, A, a_rows, a_cols, a_pitch, W, w_rows, M, N, taps, tap_off, nullptr, ep, num_sms, force_bn, false);
}

int gemm_prepare_tf32x3(GemmLaunch* out, const float* A_split, long long a_rows, int C, int C_half, const float* W3, int w_rows,
                        int M, int N, int taps, const int* tap_off, const GemmEpilogue& ep, int num_sms, int force_bn) {
  PRISMA_CHECK(taps * 3 <= GEMM_MAX_TAPS, "gemm(tf32x3): too many taps");
  PRISMA_CHECK(C % 32 == 0 && C_half % 32 == 0 && C <= C_half, "gemm(tf32x3): channel counts must be multiples of 32");
  int off[GEMM_MAX_TAPS], acol[GEMM_MAX_TAPS];
  for (int t = 0; t < taps; ++t)
    for (int p = 0; p < 3; ++p) { off[t * 3 + p] = tap_off[t]; acol[t * 3 + p] = p == 1 ? C_half : 0; }
  // external accumulation (GemmArgs::acc_group): 128-wide tiles at most (the running sums are 64 registers per thread).
  // PRISMA_TF32_ACC_GROUP=0 keeps the whole K inside one wgmma chain (the biased, cheaper variant).
  static const int acc_group = [] { const char* e = getenv("PRISMA_TF32_ACC_GROUP"); return e ? atoi(e) : 4; }();
  if (acc_group > 0 && force_bn == 0) force_bn = N > 64 ? 128 : (N > 32 ? 64 : 32);
  PRISMA_TRY(gemm_prepare_impl(out, A_split, a_rows, C, 2 * C_half, W3, w_rows, M, N, taps * 3, off, acol, ep, num_sms, force_bn, true));
  out->args.acc_group = acc_group > 0 ? acc_group : 1;
  out->xacc = acc_group > 0 && out->bn <= 128;
  return 0;
}

static int gemm_prepare_impl(GemmLaunch* out, const void* A, long long a_rows, int a_cols, int a_pitch, const void* W,
                             int w_rows, int M, int N, int taps, const int* tap_off, const int* tap_acol, const GemmEpilogue& ep_in,
                             int num_sms, int force_bn, bool tf32) {
  PRISMA_CHECK(taps >= 1 && taps <= GEMM_MAX_TAPS, "gemm: bad tap count");
  PRISMA_CHECK(N % 4 == 0, "gemm: N must be a multiple of 4");
  PRISMA_CHECK(M >= 1 && a_cols >= 1, "gemm: empty problem");
  // force_bn: 32 / 64 / 128 / 256.  512, 384 and 640 name the 256 x 256, 256 x 128 and transposed 128 x 256 tiles of the
  // sm_100 build (CTA pairs, swapped operands); Hopper has no such instructions, so they request the 256- / 128-wide tiles.
  int bn = force_bn ? force_bn : gemm_pick_bn(M, N, num_sms);
  if (bn == 512) bn = 256;
  else if (bn == 384 || bn == 640) bn = 128;
  GemmEpilogue ep = ep_in;
  // the TMA-store epilogue exists for 128- and 256-wide tiles; a problem the tile choice gives narrower tiles keeps the
  // register epilogue (same results: the TMA path is an optimisation of the same arithmetic)
  if (ep.tma_store && (bn == 32 || bn == 64) && !tf32) ep.tma_store = false;
  out->tf32 = tf32;
  out->xacc = false;
  out->args.acc_group = 1;
  const int bke = tf32 ? 32 : 64;  // elements per 128-byte K block
  PRISMA_CHECK(bn == 32 || bn == 64 || bn == 128 || bn == 256, "gemm: unsupported BLOCK_N");
  PRISMA_CHECK(w_rows >= round_up(N, bn), "gemm: weight rows must be padded to a multiple of BLOCK_N");
  const int kchunks = ceil_div(a_cols, bke);
  out->bn = bn;
  out->args.M = M;
  out->args.N = N;
  out->args.taps = taps;
  out->args.kchunks = kchunks;
  {
    static const char* r = getenv("PRISMA_GEMM_RASTER");  // "m" / "n": force (experiments)
    out->args.raster_n = r ? (r[0] == 'n') : (M >= N);
  }
  for (int t = 0; t < GEMM_MAX_TAPS; ++t) {
    out->args.tap_off[t] = t < taps ? tap_off[t] : 0;
    out->args.tap_acol[t] = (t < taps && tap_acol) ? tap_acol[t] : 0;
  }
  out->args.ep = ep;
  if (tf32) {
    // the A map spans the [hi | lo] halves (2 * a_cols columns); out-of-range columns of a ragged last K block read as zero
    PRISMA_TRY(make_tmap_2d_f32(&out->tmA, A, (uint64_t)a_pitch, (uint64_t)a_rows, (uint64_t)a_pitch, 32, GEMM_BM));
    PRISMA_TRY(make_tmap_2d_f32(&out->tmB, W, (uint64_t)taps * kchunks * 32, (uint64_t)w_rows, (uint64_t)taps * kchunks * 32, 32, bn));
  } else {
    PRISMA_TRY(make_tmap_2d_f16(&out->tmA, A, (uint64_t)a_cols, (uint64_t)a_rows, (uint64_t)a_pitch, 64, GEMM_BM));
    PRISMA_TRY(make_tmap_2d_f16(&out->tmB, W, (uint64_t)taps * kchunks * 64, (uint64_t)w_rows,
                                (uint64_t)taps * kchunks * 64, 64, bn));
  }
  const int tiles = ceil_div(M, GEMM_BM) * ceil_div(N, bn);
  out->grid = tiles < num_sms ? tiles : num_sms;
  out->flops = 2.0 * M * (double)N * taps * a_cols;
  // TMA-store epilogue: a plain dense fp32 output (scale only) leaves through swizzled shared-memory boxes and
  // cp.async.bulk.tensor stores instead of per-lane st.global (the store-bound RAFT correlation volume)
  out->tma_store = false;
  out->tmD = out->tmA;
  if (ep.tma_store) {
    PRISMA_CHECK((ep.out_f32 != nullptr) != (ep.out_f16 != nullptr) && !ep.out_f16_relu && !ep.pre_f32 && !ep.gru &&
                     !ep.res_a && !ep.res_b && ep.row_map == ROW_LINEAR && !ep.head_w && !ep.stat_part,
                 "gemm: the TMA-store epilogue handles one scaled dense output (fp32 or fp16) only");
    PRISMA_CHECK(ep.out_f16 ? (ep.act >= 0 && ep.act <= 2 && !ep.gamma && !ep.res_f32) : ep.act == 0,
                 "gemm: the TMA-store epilogue applies bias + GELU / ReLU (fp16 destinations) or bias + LayerScale (fp32) only");
    // an fp32 residual must be the destination itself (x += ...): it becomes a TMA reduce-add
    PRISMA_CHECK(!ep.res_f32 || (ep.res_f32 == ep.out_f32 && ep.res_f32_ld == ep.out_f32_ld),
                 "gemm: the TMA-store epilogue adds a residual only in place");
    out->args.ep.tma_reduce = ep.res_f32 != nullptr;
    PRISMA_CHECK(!ep.out_f16 || N % 8 == 0, "gemm: the fp16 TMA-store epilogue needs N % 8 == 0");
    PRISMA_CHECK(bn >= 128, "gemm: the TMA-store epilogue is built for BLOCK_N 128 / 256");
    if (ep.out_f16) PRISMA_TRY(make_tmap_2d_f16_store(&out->tmD, ep.out_f16, (uint64_t)N, (uint64_t)M, (uint64_t)ep.out_f16_ld));
    else PRISMA_TRY(make_tmap_2d_f32(&out->tmD, ep.out_f32, (uint64_t)N, (uint64_t)M, (uint64_t)ep.out_f32_ld, 32, 32));
    out->tma_store = true;
  }
  return 0;
}

template <int BN, bool TMAST = false, bool TF32 = false, bool XACC = false>
static int launch_bn(const GemmLaunch& g, cudaStream_t stream) {
  static bool attr_set = false;  // per-process, per-instantiation
  using Cfg = GemmCfg<BN, TMAST>;
  if (!attr_set) {
    PRISMA_CUDA_OK(cudaFuncSetAttribute(gemm_tc_kernel<BN, TMAST, TF32, XACC>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    attr_set = true;
  }
  PRISMA_CUDA_OK(pdl_launch(gemm_tc_kernel<BN, TMAST, TF32, XACC>, dim3(g.grid), dim3(GEMM_THREADS), Cfg::SMEM_BYTES, stream,
                            g.tmA, g.tmB, g.tmD, g.args));
  PRISMA_CUDA_OK(cudaGetLastError());
  return 0;
}

int gemm_run(const GemmLaunch& g, cudaStream_t stream) {
  if (g.tf32 && g.xacc) {
    switch (g.bn) {
      case 128: return launch_bn<128, false, true, true>(g, stream);
      case 64: return launch_bn<64, false, true, true>(g, stream);
      case 32: return launch_bn<32, false, true, true>(g, stream);
    }
    set_last_error("gemm_run: external accumulation needs BLOCK_N <= 128");
    return -1;
  }
  if (g.tf32) {
    switch (g.bn) {
      case 256: return launch_bn<256, false, true>(g, stream);
      case 128: return launch_bn<128, false, true>(g, stream);
      case 64: return launch_bn<64, false, true>(g, stream);
      case 32: return launch_bn<32, false, true>(g, stream);
    }
    set_last_error("gemm_run: unsupported BLOCK_N (tf32)");
    return -1;
  }
  if (g.tma_store) {
    if (g.bn == 256) return launch_bn<256, true>(g, stream);
    if (g.bn == 128) return launch_bn<128, true>(g, stream);
    set_last_error("gemm_run: no TMA-store instantiation for this tile shape");
    return -1;
  }
  switch (g.bn) {
    case 256: return launch_bn<256>(g, stream);
    case 128: return launch_bn<128>(g, stream);
    case 64: return launch_bn<64>(g, stream);
    case 32: return launch_bn<32>(g, stream);
  }
  set_last_error("gemm_run: unsupported BLOCK_N");
  return -1;
}

}  // namespace prisma
