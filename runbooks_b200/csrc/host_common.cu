#include "host_common.h"

#include <mutex>

namespace b200w {

void* DeviceMemory::alloc_bytes(size_t n) {
  const size_t bytes = (n + 255) / 256 * 256;
  void* p = nullptr;
  if (cudaMalloc(&p, bytes) != cudaSuccess) {
    cudaGetLastError();
    throw std::bad_alloc();
  }
  held_.emplace_back(p, bytes);
  bytes_ += static_cast<int64_t>(bytes);
  return p;
}

void DeviceMemory::free_held(void* p) {
  for (auto it = held_.begin(); it != held_.end(); ++it)
    if (it->first == p) {
      cudaFree(p);
      bytes_ -= static_cast<int64_t>(it->second);
      held_.erase(it);
      return;
    }
}

DeviceMemory::~DeviceMemory() {
  for (const auto& h : held_) cudaFree(h.first);
}

namespace {
using EncodeTiledFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                   const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                   const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                   CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    // libcuda is reached through the runtime: the .so carries no link-time dependency on it, so
    // it loads (and its symbols can be checked) on a box without a driver.
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q);
    if (e != cudaSuccess || q != cudaDriverEntryPointSuccess || !p)
      throw Error("cuTensorMapEncodeTiled not available from the driver");
    fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

CUtensorMap make_tmap_2d(CUtensorMapDataType type, uint32_t elem_bytes, const void* base, uint64_t rows,
                         uint64_t cols, uint64_t ld, uint32_t box_rows, uint32_t box_cols, bool swizzle) {
  B200W_CHECK((!swizzle || box_cols * elem_bytes <= 128) && box_cols <= 256 && box_rows <= 256,
              "box exceeds SWIZZLE_128B / TMA limits");
  B200W_CHECK((ld * elem_bytes) % 16 == 0, "row stride must be a multiple of 16 bytes");
  CUtensorMap m;
  cuuint64_t gdim[2] = {cols, rows};
  cuuint64_t gstride[1] = {ld * elem_bytes};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estride[2] = {1, 1};
  CUresult r = encode_fn()(&m, type, 2, const_cast<void*>(base), gdim,
                           gstride, box, estride, CU_TENSOR_MAP_INTERLEAVE_NONE,
                           swizzle ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                           CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    throw Error("cuTensorMapEncodeTiled failed with CUresult " + std::to_string((int)r));
  return m;
}
}  // namespace

CUtensorMap make_tmap_bf16_2d(const void* base, uint64_t rows, uint64_t cols, uint64_t ld,
                              uint32_t box_rows, uint32_t box_cols, bool swizzle) {
  return make_tmap_2d(CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, base, rows, cols, ld, box_rows, box_cols, swizzle);
}
CUtensorMap make_tmap_f32_2d(const void* base, uint64_t rows, uint64_t cols, uint64_t ld,
                             uint32_t box_rows, uint32_t box_cols) {
  return make_tmap_2d(CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, base, rows, cols, ld, box_rows, box_cols, true);
}
CUtensorMap make_tmap_u8_2d(const void* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows,
                            uint32_t box_cols) {
  return make_tmap_2d(CU_TENSOR_MAP_DATA_TYPE_UINT8, 1, base, rows, cols, ld, box_rows, box_cols, false);
}

int sm_count() {
  static int cache[64] = {0};
  int dev = 0;
  B200W_CUDA(cudaGetDevice(&dev));
  int& n = cache[dev & 63];
  if (!n) {
    int v = 0;
    B200W_CUDA(cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev));
    n = v;
  }
  return n;
}

namespace {
thread_local int g_sm_reserve = 0;
}
void gemm_set_sm_reserve(int n) { g_sm_reserve = n < 0 ? 0 : n; }
int gemm_sm_reserve() { return g_sm_reserve; }

}  // namespace b200w
