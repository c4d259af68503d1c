// Shared host/device declarations for libb200unet (internal; the public C ABI is include/b200unet.h).
#pragma once
#include <cstdint>
#include <cstdio>
#include <cstdarg>
#include <cstring>
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_bf16.h>

namespace b200 {

typedef __nv_bfloat16 bf16;

// Status codes returned through the C ABI.
enum Status : int { OK = 0, E_INVALID = -1, E_UNSUPPORTED = -2, E_CUDA = -3, E_DRIVER = -4 };

void set_error(const char* fmt, ...);
const char* get_error();

#define B200_CHECK_CUDA(expr)                                                                 \
  do {                                                                                        \
    cudaError_t _e = (expr);                                                                  \
    if (_e != cudaSuccess) {                                                                  \
      b200::set_error("%s:%d CUDA error %s: %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
      return b200::E_CUDA;                                                                    \
    }                                                                                         \
  } while (0)

#define B200_REQUIRE(cond, code, ...)  \
  do {                                 \
    if (!(cond)) {                     \
      b200::set_error(__VA_ARGS__);    \
      return (code);                   \
    }                                  \
  } while (0)

#define B200_TRY(expr)        \
  do {                        \
    int _s = (expr);          \
    if (_s != b200::OK) return _s; \
  } while (0)

// NDHWC bf16 tensor view.  value = hi (+ lo when lo != nullptr: split-precision "parity" mode).
struct Act {
  bf16* hi;
  bf16* lo;
  int N, D, H, W, C;  // logical extent; C = channels visible through this view
  int ld;             // channel pitch of the underlying buffer in elements (>= C)
  int vD, vH, vW;     // optional "visible" spatial extents (0 = D/H/W): voxels beyond them read as zero through TMA
  __host__ __device__ long long voxels() const { return (long long)N * D * H * W; }
};

static inline Act make_act(bf16* hi, bf16* lo, int N, int D, int H, int W, int C, int ld) {
  Act a; a.hi = hi; a.lo = lo; a.N = N; a.D = D; a.H = H; a.W = W; a.C = C; a.ld = ld; a.vD = a.vH = a.vW = 0; return a;
}
static inline Act slice_c(const Act& a, int c0, int c) {
  Act r = a; r.hi = a.hi + c0; r.lo = a.lo ? a.lo + c0 : nullptr; r.C = c; return r;
}

// Programmatic dependent launch (opt-in: B200UNET_PDL=1).  A kernel launched through launch_pdl may be scheduled while the previous
// kernel of the stream still runs: its CTAs take SMs as that kernel's CTAs retire, run their set-up (barrier init,
// descriptor prefetch) and block in pdl_wait() (ptx.cuh) until the previous kernel has completed and its writes are
// visible -- the launch latency and the set-up of every launch leave the critical path.  ONLY kernels that execute pdl_wait()
// before their first access to global memory may be launched this way.
bool pdl_enabled();

#ifdef __CUDACC__
template <typename... KArgs, typename... Args>
static inline void launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  if (!pdl_enabled()) {
    kernel<<<grid, block, smem, st>>>(args...);
    return;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = 1;
  (void)cudaLaunchKernelEx(&cfg, kernel, args...);   // the caller checks cudaGetLastError() as after a <<<>>> launch
}
#endif

// Opt Kernel in to `bytes` of dynamic shared memory, once per device: not a stream operation, so it stays out of CUDA-graph
// captures after the first launch.  Keyed by the kernel itself (instantiations of one template share a signature).
template <auto Kernel>
static inline int set_max_dynamic_smem(int bytes) {
  static bool done[64] = {};
  int dev = 0;
  B200_CHECK_CUDA(cudaGetDevice(&dev));
  if (dev >= 64 || !done[dev]) {
    B200_CHECK_CUDA(cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    if (dev < 64) done[dev] = true;
  }
  return OK;
}

// SMs of the current device; 132 (an H100 SXM) on a host without a GPU (route queries, planning).
inline int device_sms() {
  int dev = 0, sms = 0;
  if (cudaGetDevice(&dev) == cudaSuccess && cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && sms > 0)
    return sms;
  cudaGetLastError();
  return 132;
}

static inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
static inline int round_up(int a, int b) { return ceil_div(a, b) * b; }

}  // namespace b200
