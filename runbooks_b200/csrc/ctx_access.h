// Narrow window onto b200w_ctx (defined in engine.cu) for the other translation units.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/b200w.h"
#include "host_common.h"

struct b200w_ctx;

int ctx_device(b200w_ctx* c);
cudaStream_t ctx_stream(b200w_ctx* c);
void ctx_set_error(b200w_ctx* c, const char* msg);
int64_t& ctx_launches(b200w_ctx* c);
void* ctx_infer_slot(b200w_ctx* c);
void ctx_set_infer(b200w_ctx* c, void* p, void (*destroy)(void*));
// normal(0, std) / constant fill of a bf16 range with the engine's counter-based generator
// element j of w_bf16 gets the value of flat index i0 + j of the seeded fill
void ctx_fill_normal(b200w_ctx* c, void* w_bf16, size_t n, uint64_t seed, float std, size_t i0 = 0);
void ctx_fill_const(b200w_ctx* c, void* w_bf16, size_t n, float value);
// 8 floats of device scratch for the per-kernel hooks, allocated from the context's memory at first use
float* ctx_scal(b200w_ctx* c);

// Called from a catch (...) block: rethrows the exception in flight, records its message as the context's error and
// returns its status. NcclError: B200W_ERR_NCCL; std::bad_alloc: B200W_ERR_OOM; InvalidArgument: B200W_ERR_INVALID;
// StateError: B200W_ERR_STATE; any other Error: B200W_ERR_CUDA; any other std::exception: B200W_ERR_INVALID. An
// NCCL or CUDA failure also marks the context dead, so that b200w_destroy aborts its communicator.
int ctx_fail(b200w_ctx* c);

// The body of a C entry point: f() on the context's device, its exceptions turned into a status by ctx_fail.
// A NULL context is B200W_ERR_INVALID.
template <typename F>
int guarded(b200w_ctx* ctx, F&& f) {
  if (!ctx) return B200W_ERR_INVALID;
  try {
    B200W_CUDA(cudaSetDevice(ctx_device(ctx)));
    f();
    return B200W_OK;
  } catch (...) {
    return ctx_fail(ctx);
  }
}
