// Host-side plumbing shared by the kernel launchers: error capture, memory ownership and TMA tensor-map creation.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <memory>
#include <mutex>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include <nvtx3/nvToolsExt.h>

namespace b200w {

// The exceptions the library throws. ctx_fail (ctx_access.h) turns each into the status named here, by type alone.
// a failed CUDA call or a broken internal invariant (B200W_ERR_CUDA; the context is dead)
struct Error : std::runtime_error {
  using std::runtime_error::runtime_error;
};
// an argument the call refuses (B200W_ERR_INVALID); B200W_CHECK throws it
struct InvalidArgument : std::runtime_error {
  using std::runtime_error::runtime_error;
};
// a call that does not fit the context's configuration or the calls before it (B200W_ERR_STATE)
struct StateError : std::runtime_error {
  using std::runtime_error::runtime_error;
};

#define B200W_CUDA(expr)                                                                   \
  do {                                                                                     \
    cudaError_t _e = (expr);                                                               \
    if (_e != cudaSuccess)                                                                 \
      throw ::b200w::Error(std::string(#expr) + " failed: " + cudaGetErrorString(_e) +     \
                           " (" __FILE__ ":" + std::to_string(__LINE__) + ")");            \
  } while (0)

#define B200W_CHECK(cond, msg)                                                             \
  do {                                                                                     \
    if (!(cond))                                                                           \
      throw ::b200w::InvalidArgument(std::string("check failed: " #cond " — ") + (msg) +   \
                                     " (" __FILE__ ":" + std::to_string(__LINE__) + ")");  \
  } while (0)

// The device memory a context holds: each allocation is cudaMalloc'd in whole 256-byte units, and bytes() is the sum
// of the units currently held. release and the destructor free with cudaFree, which waits for the device, so a
// buffer that enqueued work still reads may be released.
class DeviceMemory {
 public:
  DeviceMemory() = default;
  DeviceMemory(const DeviceMemory&) = delete;
  DeviceMemory& operator=(const DeviceMemory&) = delete;
  ~DeviceMemory();
  // n elements of T; std::bad_alloc, with the CUDA error cleared, when the device has no room
  template <typename T>
  T* alloc(size_t n) {
    return static_cast<T*>(alloc_bytes(n * sizeof(T)));
  }
  // frees p, takes its bytes off the count and sets p to nullptr; a pointer alloc did not return (nullptr
  // included) is only cleared
  template <typename T>
  void release(T*& p) {
    free_held(p);
    p = nullptr;
  }
  int64_t bytes() const { return bytes_; }

 private:
  void* alloc_bytes(size_t n);
  void free_held(void* p);
  std::vector<std::pair<void*, size_t>> held_;
  int64_t bytes_ = 0;
};

struct CudaFree {
  void operator()(void* p) const { cudaFree(p); }
};
struct CudaFreeHost {
  void operator()(void* p) const { cudaFreeHost(p); }
};

// Device scratch for the length of one call, counted by no DeviceMemory: n elements of T, freed with cudaFree when
// it goes out of scope. A failed cudaMalloc throws Error, as every failed CUDA call does.
template <typename T>
using DeviceScratch = std::unique_ptr<T[], CudaFree>;
template <typename T>
DeviceScratch<T> device_scratch(size_t n) {
  void* p = nullptr;
  B200W_CUDA(cudaMalloc(&p, n * sizeof(T)));
  return DeviceScratch<T>(static_cast<T*>(p));
}

// Pinned host memory: n elements of T from cudaMallocHost, freed with cudaFreeHost. To regrow one, reset() it before
// allocating the new one, so that the two are never held at once.
template <typename T>
using PinnedBuffer = std::unique_ptr<T[], CudaFreeHost>;
template <typename T>
PinnedBuffer<T> pinned_buffer(size_t n) {
  void* p = nullptr;
  B200W_CUDA(cudaMallocHost(&p, n * sizeof(T)));
  return PinnedBuffer<T>(static_cast<T*>(p));
}

// ceil(a / b) for a grid size
inline int cdiv(long long a, int b) { return static_cast<int>((a + b - 1) / b); }

// 2-D bf16 row-major tensor [rows, cols] with leading dimension ld (elements).
// Box = [box_rows, box_cols], each at most 256; box_cols * 2 bytes must be <= 128 (SWIZZLE_128B span) when swizzled.
// Out-of-bounds elements are zero-filled by the hardware (used for K / M / N tails).
// swizzle = false: the box is stored in shared memory as plain rows (no SWIZZLE_128B permutation).
CUtensorMap make_tmap_bf16_2d(const void* base, uint64_t rows, uint64_t cols, uint64_t ld,
                              uint32_t box_rows, uint32_t box_cols, bool swizzle = true);
// The same for fp32 elements (box_cols * 4 bytes <= 128).
CUtensorMap make_tmap_f32_2d(const void* base, uint64_t rows, uint64_t cols, uint64_t ld,
                             uint32_t box_rows, uint32_t box_cols);

// 2-D byte tensor (e4m3 KV cache) [rows, cols], stored in shared memory as plain rows (box_cols a multiple of 16).
CUtensorMap make_tmap_u8_2d(const void* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows,
                            uint32_t box_cols);

// SM count of the CURRENT device (cached per device: a process may hold contexts on several GPUs)
int sm_count();

// First-use work that is per DEVICE, not per process: cudaFuncSetAttribute(MaxDynamicSharedMemorySize)
// applies to the current device only, so a process-wide `static bool` breaks the second GPU of a
// one-process-many-contexts host (INTEGRATION.md's cgo layout).
//   static PerDeviceOnce once; once.run([&] { cudaFuncSetAttribute(...); });
class PerDeviceOnce {
 public:
  template <typename F>
  void run(F&& f) {
    int dev = 0;
    B200W_CUDA(cudaGetDevice(&dev));
    const uint64_t bit = 1ull << (dev & 63);
    std::lock_guard<std::mutex> lock(mu_);
    if (done_ & bit) return;
    f();
    done_ |= bit;
  }

 private:
  std::mutex mu_;
  uint64_t done_ = 0;
};

// Kernel launch with the programmatic-stream-serialization attribute (see ptx.cuh pdl_wait): only for
// kernels that call pdl_wait() before they touch anything their predecessor wrote.
// cluster_y > 1 additionally groups that many consecutive blockIdx.y CTAs into a thread-block cluster.
template <typename... KArgs, typename... Args>
void launch_pdl_cluster(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, int cluster_y,
                        Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = s;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  int n = 1;
  if (cluster_y > 1) {
    attr[1].id = cudaLaunchAttributeClusterDimension;
    attr[1].val.clusterDim.x = 1;
    attr[1].val.clusterDim.y = static_cast<unsigned>(cluster_y);
    attr[1].val.clusterDim.z = 1;
    n = 2;
  }
  cfg.attrs = attr;
  cfg.numAttrs = n;
  B200W_CUDA(cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(std::forward<Args>(args))...));
}
template <typename... KArgs, typename... Args>
void launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, Args&&... args) {
  launch_pdl_cluster(kern, grid, block, smem, s, 1, std::forward<Args>(args)...);
}

// NVTX range for the phases of a step (header-only NVTX v3: a no-op costing one predictable branch unless a tool
// such as nsys / ncu --nvtx is attached). SURVEY.md 5, tracing row.
struct NvtxRange {
  explicit NvtxRange(const char* name) { nvtxRangePushA(name); }
  ~NvtxRange() { nvtxRangePop(); }
  NvtxRange(const NvtxRange&) = delete;
  NvtxRange& operator=(const NvtxRange&) = delete;
};

// gemm_bf16 leaves this many SMs free (grid = SMs - reserve): set around the backward that runs
// concurrently with the NCCL gradient all-reduce, so that NCCL's CTAs find SMs without waiting for a
// persistent GEMM CTA to end and the GEMM's CTAs never queue behind NCCL's. Per host thread.
void gemm_set_sm_reserve(int n);
int gemm_sm_reserve();

}  // namespace b200w
