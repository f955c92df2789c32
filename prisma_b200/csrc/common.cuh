// prisma_b200 -- common device/host helpers for sm_90a (H100).
// Hand-written PTX wrappers for mbarrier, TMA (cp.async.bulk.tensor), warpgroup MMA descriptors.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <string>

namespace prisma {

// ----------------------------------------------------------------------------------------------
// host-side error plumbing: nothing throws across the C ABI; errors become codes + thread-local text
// ----------------------------------------------------------------------------------------------
void set_last_error(const std::string& msg);

#define PRISMA_CUDA_OK(expr)                                                                     \
  do {                                                                                           \
    cudaError_t _e = (expr);                                                                     \
    if (_e != cudaSuccess) {                                                                     \
      ::prisma::set_last_error(std::string(#expr) + " failed: " + cudaGetErrorString(_e) +       \
                               " (" __FILE__ ":" + std::to_string(__LINE__) + ")");              \
      return -2;                                                                                 \
    }                                                                                            \
  } while (0)

#define PRISMA_CHECK(cond, msg)                                                                  \
  do {                                                                                           \
    if (!(cond)) {                                                                               \
      ::prisma::set_last_error(std::string(msg) + " [" #cond "] (" __FILE__ ":" +                \
                               std::to_string(__LINE__) + ")");                                  \
      return -1;                                                                                 \
    }                                                                                            \
  } while (0)

#define PRISMA_TRY(expr)                                                                         \
  do {                                                                                           \
    int _r = (expr);                                                                             \
    if (_r != 0) return _r;                                                                      \
  } while (0)

// NVTX ranges (header-only nvtx3: a no-op unless a profiler injects its library) around every engine pass and, in the
// un-graphed direct runs, around every named step -- so an Nsight Systems / ncu --nvtx timeline reads in the reference's
// vocabulary (SURVEY.md section 5: the reference has no tracing hooks at all).
struct NvtxRange {
  explicit NvtxRange(const char* name);
  ~NvtxRange();
};

static inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
static inline int round_up(int a, int b) { return ceil_div(a, b) * b; }

#ifdef __CUDACC__
// ----------------------------------------------------------------------------------------------
// device helpers
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t.reg .pred P;\n\telect.sync _|P, 0xffffffff;\n\tselp.b32 %0, 1, 0, P;\n\t}\n"
      : "=r"(pred));
  return pred != 0;
}

// ---- programmatic dependent launch ------------------------------------------------------------------
// Every kernel of a band's pass begins with pdl_prologue(): (1) griddepcontrol.launch_dependents lets the NEXT kernel of the
// stream / graph be scheduled as soon as every CTA of this one has started -- its CTAs become resident where resources
// allow, run their own prologue (barrier init, descriptor prefetch) and block in (2) griddepcontrol.wait,
// which returns when the PREVIOUS kernel has completed and its writes are visible.  Nothing touches global memory before
// the wait, so the dependency chain is the stream order, only the ~2-4 us of launch latency and prologue per kernel
// overlap the predecessor's tail (a RAFT pass is ~330 kernels of 5-40 us).  Both instructions are no-ops for a kernel
// launched without the programmatic-serialization attribute (pdl_launch below sets it).
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_prologue() { pdl_launch_dependents(); pdl_wait(); }

// ---- mbarrier ---------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug becomes a trap (-> CUDA error on the host), never a hung GPU.  No printf here: a function
// call inside a wgmma kernel makes ptxas serialise its wgmma pipeline.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 4000000000LL) __trap();  // ~2 s
  }
}

// ---- TMA ----------------------------------------------------------------------------------------
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}

// TMA store: a swizzled shared-memory box -> global (bulk async group of the issuing thread); out-of-range rows / columns
// of the box are clipped by the tensor map
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void tma_store_wait_read() {  // at most N groups of this thread still READING shared memory
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// ---- warpgroups -------------------------------------------------------------------------------------
// register re-allocation between the producer and the consumer warpgroups of a warp-specialised kernel
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
// named barrier over `count` threads (id 0 is __syncthreads)
__device__ __forceinline__ void named_bar_sync(int id, int count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}

// wgmma shared-memory matrix descriptor, 128B-swizzled tiles whose rows are 128 bytes (64 fp16 / 32 fp32):
//   K-major  : rows = M/N index, 8-row groups 1024 B apart (SBO); K advances inside the 128 B row (+32 B = +2 per K step).
//   MN-major : rows = K index, 128 B = 64 MN elements; 8-row K groups 1024 B apart (SBO).
// Fields (PTX ISA, "Matrix Descriptor Format" of wgmma): addr>>4 [0,14) | LBO>>4 [16,30) | SBO>>4 [32,46) |
// base offset [49,52) = 0 (1024-aligned tiles) | layout_type [62,64) (1 = SWIZZLE_128B).
__device__ __forceinline__ uint64_t make_wgmma_desc(uint32_t smem_addr, uint32_t sbo_bytes = 1024, uint32_t lbo_bytes = 16) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}

// ---- misc math ------------------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_min(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fminf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ uint32_t pack_half2(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}
#endif  // __CUDACC__

// ----------------------------------------------------------------------------------------------
// host: TMA descriptor encode through the runtime's driver entry point (no -lcuda link dependency)
// ----------------------------------------------------------------------------------------------
// 2-D fp16 tensor [rows][cols] with row pitch `pitch_elems`; box = box_cols x box_rows, 128B swizzle
// (box_cols must be 64 -> 128-byte inner box).  Out-of-bounds elements (either sign) read as zero.
int make_tmap_2d_f16(CUtensorMap* out, const void* base, uint64_t cols, uint64_t rows, uint64_t pitch_elems,
                     uint32_t box_cols, uint32_t box_rows);
// the same for an fp32 tensor (box_cols must be 32 -> 128-byte inner box): the destination of the TMA-store epilogue
int make_tmap_2d_f32(CUtensorMap* out, const void* base, uint64_t cols, uint64_t rows, uint64_t pitch_elems,
                     uint32_t box_cols, uint32_t box_rows);

// SM count of the current device (cached per device): the grid size of the grid-stride pointwise kernels is a small multiple
// of it, so every SM gets the same number of resident blocks.
int device_sm_count();

// Launch with the programmatic-stream-serialization attribute when PRISMA_PDL=1 (default: a plain launch; see gemm.cu for the
// measurement that turned it off).
bool pdl_enabled();
#ifdef __CUDACC__
template <typename... KArgs, typename... Args>
inline cudaError_t pdl_launch(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = s;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}
#endif

}  // namespace prisma
